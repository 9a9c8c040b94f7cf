"""Evaluation without a GPU: the float64 reduction of episode records (rlca_eval_reduce_host runs the device code's
per-world function on the CPU), the metric definitions of DESIGN.md §9c, and the circle layouts."""
import math

import numpy as np
import pytest

from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

DT, GOAL_R, VMAX = 0.1, 0.5, 1.0


def _cfg(worlds, robots):
    sc = make_scenario('stage1', robots_per_world=robots)
    return fill_config(_lib.EnvConfig(), sc, num_worlds=worlds, beams=512)


def _reduce(records, count, open_, worlds, world_begin=0, world_count=None):
    from rl_collision_avoidance_b200.evaluation import reduce_host
    return reduce_host(_cfg(worlds, records.shape[0] // worlds), records, count, open_, world_begin, world_count)


def test_eval_symbols_exported(built):
    lib = _lib.load()
    for n in ('rlca_eval_track', 'rlca_eval_reduce', 'rlca_eval_reduce_host'):
        assert hasattr(lib, n) and n in _lib.SYMBOLS
    assert len(_lib.EVAL_PARTIALS) == 14


def test_metrics_on_hand_made_records(built):
    """Known answers: two worlds of two robots, E = 2.  World 0: a 3.0 m start-goal distance reached in 40 ticks along a
    3.2 m path, a goal 0.3 m away (L clamped to 0) reached in 5 ticks along 0.25 m, one crash, one time-out.  World 1:
    nothing reached, one crash and an unfinished robot (no record, in an episode)."""
    from rl_collision_avoidance_b200.evaluation import metrics, totals
    f32 = np.float32
    rec = np.zeros((4, 2, 4), np.float32)
    rec[0, 0] = (1, 40, 3.2, 3.0)
    rec[0, 1] = (2, 7, 0.7, 2.0)
    rec[1, 0] = (1, 5, 0.25, 0.3)
    rec[1, 1] = (3, 151, 9.0, 4.0)
    rec[2, 0] = (2, 12, 1.1, 5.0)
    count = np.array([2, 2, 1, 0], np.int32)
    open_ = np.array([1, 1, 0, 1], np.int32)
    p = _reduce(rec, count, open_, worlds=2)
    dt = float(f32(DT))                                      # the config's fp32 dt
    T1, T2 = 40 * dt, 5 * dt
    L1, L2 = float(f32(3.0)) - GOAL_R, 0.0
    P1, P2 = float(f32(3.2)), float(f32(0.25))
    et = (T1 - L1 / VMAX, T2 - L2 / VMAX)
    ed = (P1 - L1, P2 - L2)
    sp = (P1 / T1, P2 / T2)
    assert p.shape == (2, 14)
    assert list(p[0, :4]) == [2, 1, 1, 0] and list(p[1, :4]) == [0, 1, 0, 1]
    assert p[0, 4] == pytest.approx(T1 + T2) and p[0, 5] == pytest.approx(T1 ** 2 + T2 ** 2)
    assert p[0, 6] == pytest.approx(sum(et)) and p[0, 7] == pytest.approx(sum(x * x for x in et))
    assert p[0, 8] == pytest.approx(sum(ed)) and p[0, 9] == pytest.approx(sum(x * x for x in ed))
    assert p[0, 10] == pytest.approx(sum(sp)) and p[0, 11] == pytest.approx(sum(x * x for x in sp))
    assert p[0, 12] == pytest.approx(float(f32(3.0)) + float(f32(0.3))) and p[0, 13] == pytest.approx(P1 + P2)
    assert np.all(p[1, 4:] == 0)                             # the all-failed world contributes no sums
    m = metrics(totals(p))
    assert (m['episodes'], m['reached'], m['crashed'], m['timed_out'], m['unfinished']) == (5, 2, 2, 1, 1)
    assert m['success_rate'] == pytest.approx(0.4) and m['crash_rate'] == pytest.approx(0.4)
    assert m['extra_distance'][0] == pytest.approx(np.mean(ed)) and m['extra_distance'][1] == pytest.approx(np.std(ed))
    assert m['extra_time'][0] == pytest.approx(np.mean(et)) and m['extra_time'][1] == pytest.approx(np.std(et))
    assert m['average_speed'][0] == pytest.approx(np.mean(sp)) and m['average_speed'][1] == pytest.approx(np.std(sp))
    assert m['extra_time'][0] == pytest.approx(((4.0 - 2.5) + 0.5) / 2)
    failed = metrics(totals(p[1:]))
    assert failed['success_rate'] == 0.0 and all(math.isnan(x) for x in failed['extra_time'])


def _numpy_partials(rec, count, open_, worlds, E):
    """The definitions of DESIGN.md §9c in numpy float64, summed in the kernel's order (agent, then record)."""
    R = rec.shape[0] // worlds
    dt = float(np.float32(DT))
    out = np.zeros((worlds, 14))
    for w in range(worlds):
        s = out[w]
        for a in range(w * R, (w + 1) * R):
            c = int(count[a])
            if c < E and open_[a]:
                s[3] += 1.0
            for i in range(min(c, E)):
                res, ticks, path, D = (float(x) for x in rec[a, i])
                if res != 1:
                    s[{2: 1, 3: 2}[int(res)]] += 1.0
                    continue
                T = ticks * dt
                L = max(D - GOAL_R, 0.0)
                for k, m in enumerate((T, T - L / VMAX, path - L, path / T)):
                    s[4 + 2 * k] += m
                    s[5 + 2 * k] += m * m
                s[0] += 1.0
                s[12] += D
                s[13] += path
    return out


def test_reduction_against_numpy(built):
    """Random records of 7 worlds x 24 robots x E = 3: partials bit-equal to the float64 numpy sums in the same order,
    any world range reduces to the same rows, and the totals are a left-to-right sum of the rows."""
    from rl_collision_avoidance_b200.evaluation import totals
    rng = np.random.default_rng(3)
    W, R, E = 7, 24, 3
    N = W * R
    rec = np.zeros((N, E, 4), np.float32)
    rec[..., 0] = rng.choice([1, 1, 1, 2, 3], size=(N, E))
    rec[..., 1] = rng.integers(1, 152, size=(N, E))
    rec[..., 3] = rng.uniform(0.0, 12.0, size=(N, E))
    rec[..., 2] = rec[..., 3] * rng.uniform(0.9, 2.0, size=(N, E))
    count = rng.integers(0, 5, size=N).astype(np.int32)
    open_ = rng.integers(0, 2, size=N).astype(np.int32)
    p = _reduce(rec, count, open_, W)
    ref = _numpy_partials(rec, count, open_, W, E)
    assert np.array_equal(p.view(np.uint64), ref.view(np.uint64))
    assert np.array_equal(_reduce(rec, count, open_, W, 2, 3), p[2:5])
    tot = totals(p)
    acc = np.zeros(14)
    for row in ref:
        acc = acc + row
    assert np.array_equal(tot, acc)
    assert np.allclose(tot, ref.sum(0), rtol=1e-12)


def test_reduce_rejects_bad_ranges(built):
    from rl_collision_avoidance_b200.evaluation import reduce_host
    cfg = _cfg(2, 24)
    z = np.zeros((48, 1, 4), np.float32)
    zi = np.zeros(48, np.int32)
    for wb, wc in ((-1, 1), (0, 3), (2, 1), (1, 0)):
        with pytest.raises(_lib.RlcaError):
            reduce_host(cfg, z, zi, zi, wb, wc)


def _wrap(a):
    return np.remainder(a + np.pi, 2 * np.pi) - np.pi


def test_circle_layout_reproduces_the_shipped_table():
    ship = make_scenario('circle')
    sc = make_scenario('circle', robots_per_world=50, radius=25.0)
    assert sc.robots_per_world == 50 and sc.init_tab.shape == (50, 4) and sc.goal_tab.shape == (50, 4)
    assert np.abs(sc.init_tab[:, :2] - ship.init_tab[:, :2]).max() <= 0.006
    assert np.abs(sc.goal_tab[:, :2] - ship.goal_tab[:, :2]).max() <= 0.006
    assert np.abs(_wrap(sc.init_tab[:, 2].astype(np.float64) - ship.init_tab[:, 2])).max() <= 1e-6
    assert np.all(sc.init_tab[:, 2] > -np.pi) and np.all(sc.init_tab[:, 2] <= np.pi)
    assert np.all(sc.init_tab[:, 3] == 0) and np.all(sc.goal_tab[:, 2:] == 0)
    # the defaults keep the shipped table itself
    for s in (make_scenario('circle', robots_per_world=50), make_scenario('circle', robots_per_world=None)):
        assert np.array_equal(s.init_tab, ship.init_tab) and np.array_equal(s.goal_tab, ship.goal_tab)


@pytest.mark.parametrize('K,r', [(2, 5.0), (12, 10.0), (64, 25.0), (64, 5.0), (24, 12.0)])
def test_circle_layout_geometry(K, r):
    sc = make_scenario('circle', robots_per_world=K, radius=r)
    a = 2 * np.pi * np.arange(K) / K
    assert sc.robots_per_world == K
    assert np.allclose(sc.init_tab[:, 0], r * np.cos(a), atol=1e-5) and np.allclose(sc.init_tab[:, 1], r * np.sin(a), atol=1e-5)
    assert np.allclose(sc.goal_tab[:, :2], -sc.init_tab[:, :2])
    assert np.abs(_wrap(sc.init_tab[:, 2] - (np.pi + a))).max() < 1e-6


@pytest.mark.parametrize('K,r,what', [(1, 10.0, '2..64'), (65, 25.0, '2..64'), (64, 3.0, 'overlap'),
                                      (40, 2.0, 'overlap'), (12, 31.0, 'free cells'), (12, 29.9, 'free cells'),
                                      (12, 0.0, 'radius')])
def test_circle_layout_rejects(K, r, what):
    with pytest.raises(ValueError, match=what):
        make_scenario('circle', robots_per_world=K, radius=r)


def test_circle_world_accepts_num_env():
    """circle_world.StageWorld builds the K-robot scenario (the constructor then needs a GPU)."""
    import torch
    from rl_collision_avoidance_b200.circle_world import StageWorld
    if torch.cuda.is_available():
        env = StageWorld(512, num_env=12, radius=10.0)
        assert env.num_env == 12 and env.N == 12
        return
    with pytest.raises(_lib.RlcaError):
        StageWorld(512, num_env=12, radius=10.0)
    with pytest.raises(ValueError):
        StageWorld(512, num_env=70)
