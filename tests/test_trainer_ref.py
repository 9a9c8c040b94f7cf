"""The restatement of the reference's training loop (tests/trainer_ref.py) against hand-worked answers, and the host
helpers the trainer shares with it.  No GPU needed."""
import numpy as np
import pytest
import torch

import trainer_ref as ref


def test_scan_deque_starts_with_three_copies_and_shifts():
    a, b, c, d = (np.full(4, k, np.float32) for k in range(4))
    s = ref.Stacks(np.stack([a, a]))
    s.tick(np.stack([b, b]), restart=[False, False])
    s.tick(np.stack([c, d]), restart=[False, True])
    got = s.array()
    assert np.array_equal(got[0], np.stack([a, b, c]))          # popleft / append
    assert np.array_equal(got[1], np.stack([d, d, d]))          # a new episode: [obs] * 3
    s.tick(np.stack([a, b]), restart=[False, False])
    assert np.array_equal(s.array()[1], np.stack([d, d, b]))


def test_run_of_dones_crosses_a_column_boundary():
    """Column 0 ends on two dones and column 1 starts with one: the counter carries it to 3, so row (t=0, i=1) is
    filtered although it is the first done of its column.  By hand (num_env * j + i): (j=2, i=0) -> 4, (0, 1) -> 1."""
    d = np.array([[False, True],
                  [True, False],
                  [True, True]])
    assert ref.filter_index(d) == [4, 1]
    from rl_collision_avoidance_b200.model.utils import get_filter_index
    assert get_filter_index(d) == [4, 1]
    assert get_filter_index(torch.from_numpy(d)) == [4, 1]
    # no carry without the leak: the same columns side by side with a false row between them filter only (2, 0)
    assert ref.filter_index(np.array([[False, True], [True, False], [True, True], [False, False]])) == [4]


def test_idle_stage2_robot_keeps_its_stale_reward_in_the_normalised_advantages():
    """Robot 0 ends its episode on tick 0 with r = 1 and idles for ticks 1 and 2; robot 1 is live with r = 0.
    gamma 0.5, lambda 1, values and last value 0.  Robot 0's rows are (1, T), (1, T), (1, T) (the stale r), so its
    advantages are 1, 1, 1 and robot 1's 0, 0, 0: mean 1/2, population std 1/2, normalised +1 and -1.  Rows 2 and 4
    (robot 0's idle ticks) are filtered; the kept rows 0, 1, 3, 5 hold +1, -1, -1, -1.  With a zero reward on the idle
    ticks the kept rows of robot 1 would be -1/sqrt(5) = -0.447, and with the normalisation after np.delete
    -1/sqrt(3) = -0.577."""
    rows0 = ref.liveflag_rows([(1.0, True)], 3)
    assert rows0 == [(1.0, True)] * 3
    rows1 = ref.liveflag_rows([(0.0, False)] * 3, 3)
    r = np.array([[a[0], b[0]] for a, b in zip(rows0, rows1)])
    d = np.array([[a[1], b[1]] for a, b in zip(rows0, rows1)])
    tg, adv = ref.gae(r, np.zeros((3, 2)), np.zeros(2), d, 0.5, 1.0)
    assert np.array_equal(adv, [[1, 0], [1, 0], [1, 0]])
    fi = ref.filter_index(d)
    assert fi == [2, 4]
    keep = ref.kept_rows(6, fi)
    assert keep.tolist() == [0, 1, 3, 5]
    assert np.allclose(ref.normalise(adv).reshape(-1)[keep], [1, -1, -1, -1], rtol=0, atol=1e-15)
    fresh = np.array([[1, 0], [0, 0], [0, 0]], np.float64)          # what a reward of 0 on idle ticks would give
    assert np.isclose(ref.normalise(fresh).reshape(-1)[keep][1], -1 / np.sqrt(5), rtol=0, atol=1e-15)
    after = ref.normalise(adv.reshape(-1)[keep])
    assert np.isclose(after[1], -1 / np.sqrt(3), rtol=0, atol=1e-15)


def test_liveflag_rows_of_a_robot_that_ends_last():
    rows = ref.liveflag_rows([(0.5, False), (-2.0, False), (15.0, True)], 3)
    assert rows == [(0.5, False), (-2.0, False), (15.0, True)]


def test_horizon_ending_on_a_terminal_tick_masks_the_last_value():
    """H = 2, one robot: rewards 1, 2, values 0.5, 0.25, gamma 0.9, lambda 0.8, last value 100.
    Terminal last tick: delta_1 = 2 - 0.25 = 1.75 (the last value masked); delta_0 = 1 + 0.9 * 0.25 - 0.5 = 0.725;
    gae_0 = 0.725 + 0.72 * 1.75 = 1.985; targets 2.485, 2.0.  Without the terminal: delta_1 = 2 + 90 - 0.25 = 91.75,
    gae_0 = 0.725 + 0.72 * 91.75 = 66.785."""
    r, v = np.array([[1.0], [2.0]]), np.array([[0.5], [0.25]])
    tg, adv = ref.gae(r, v, [100.0], np.array([[0], [1]]), 0.9, 0.8)
    assert np.allclose(adv[:, 0], [1.985, 1.75], rtol=0, atol=1e-13)
    assert np.allclose(tg[:, 0], [2.485, 2.0], rtol=0, atol=1e-13)
    _, adv = ref.gae(r, v, [100.0], np.array([[0], [0]]), 0.9, 0.8)
    assert np.allclose(adv[:, 0], [66.785, 91.75], rtol=0, atol=1e-12)
    # a terminal first tick cuts the recurrence: row 0 is r - v alone
    _, adv = ref.gae(r, v, [100.0], np.array([[1], [0]]), 0.9, 0.8)
    assert adv[0, 0] == 0.5


def test_ragged_minibatch_and_dropped_tail():
    perm = np.array([7, 2, 9, 0, 4, 8, 1, 6, 3, 5])
    stage1 = ref.minibatches(perm, 4, drop_last=False)
    assert [b.tolist() for b in stage1] == [[7, 2, 9, 0], [4, 8, 1, 6], [3, 5]]
    stage2 = ref.minibatches(perm, 4, drop_last=True)
    assert [b.tolist() for b in stage2] == [[7, 2, 9, 0], [4, 8, 1, 6]]
    assert len(ref.minibatches(perm, 5, drop_last=True)) == 2        # an exact multiple drops nothing
    # the schedule of torch's own BatchSampler over the same order
    from torch.utils.data.sampler import BatchSampler
    for drop in (False, True):
        want = list(BatchSampler(perm.tolist(), 4, drop_last=drop))
        assert [b.tolist() for b in ref.minibatches(perm, 4, drop)] == want


def test_adam_first_step_by_hand():
    """Step 1 from zero moments: m = 0.1 g, v = 0.001 g^2, the bias corrections make them g and g^2, so
    p' = p - lr g / (|g| + eps)."""
    p, g = np.array([1.0, -2.0, 0.5]), np.array([0.3, -1e-3, 0.0])
    p1, m1, v1 = ref.adam_step(p, g, np.zeros(3), np.zeros(3), 1, 5e-5)
    assert np.allclose(m1, 0.1 * g, rtol=1e-15, atol=0)
    assert np.allclose(v1, 0.001 * g * g, rtol=1e-12, atol=0)
    assert np.allclose(p1, p - 5e-5 * g / (np.abs(g) + 1e-8), rtol=1e-14, atol=0)


def test_adam_equals_torch_optim_adam_in_float64():
    rs = np.random.RandomState(3)
    p0 = rs.standard_normal(64)
    pt = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([pt], lr=5e-5)
    p, m, v = p0.copy(), np.zeros(64), np.zeros(64)
    for step in range(1, 8):
        g = rs.standard_normal(64) * 10.0 ** rs.uniform(-6, 0, 64)
        pt.grad = torch.from_numpy(g.copy())
        opt.step()
        p, m, v = ref.adam_step(p, g, m, v, step, 5e-5)
        st = opt.state[pt]
        # torch forms m as a lerp, m + (1 - b1) (g - m): the two agree to a few float64 roundings of |m| + |g|
        assert np.abs(st['exp_avg'].numpy() - m).max() <= 1e-15 * np.abs(g).max() * step
        assert np.allclose(st['exp_avg_sq'].numpy(), v, rtol=1e-14, atol=0)
        assert np.allclose(pt.detach().numpy(), p, rtol=0, atol=1e-15)


@pytest.mark.parametrize('T,N', [(5, 3), (8, 1), (1, 7)])
def test_product_filter_index_equals_the_loop(T, N):
    from rl_collision_avoidance_b200.model.utils import get_filter_index
    rs = np.random.RandomState(T * 10 + N)
    for _ in range(50):
        d = rs.rand(T, N) < 0.6
        assert get_filter_index(d) == ref.filter_index(d)
