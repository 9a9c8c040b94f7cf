"""Non-cooperative robots without a GPU (DESIGN.md §9h): rlca_noncoop_action_host against ORCA-DD's action for an
agent without neighbours and against a float64 restatement, rlca_eval_reduce_split_host against numpy, the evaluation
helpers, the command-line checks, and the register budget of both new kernels."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import orca_ref
from helpers import make_pair, random_actions
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.evaluation import AUTO_RESET, NPARTIALS
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _states(scenario, worlds, ticks, seed):
    """EnvConfig and (pose, goal, meta) of the CPU oracle after `ticks` random-action ticks."""
    sc, _, orc = make_pair(scenario, num_worlds=worlds, gpu=False, seed=seed, auto_reset=AUTO_RESET[scenario])
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(seed)
    for _ in range(ticks):
        orc.step(random_actions(rng, orc.N))
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=worlds, beams=512, auto_reset=AUTO_RESET[scenario], seed=seed)
    return cfg, orc.pose.copy(), orc.goal.copy(), orc.meta.copy()


STATES = [('stage1', 3, 12, 1), ('stage2', 2, 12, 2), ('circle', 1, 12, 3)]


def _sentinel(rng, n):
    act = rng.uniform(-5, 5, (n, 2)).astype(np.float32)
    act[::7, 0] = np.nan
    return act


@pytest.mark.parametrize('scenario,worlds,ticks,seed', STATES)
def test_full_speed_equals_orca_dd_without_neighbours(built, scenario, worlds, ticks, seed):
    """speed = v_max: the driver's action is ORCA-DD's with a neighbour distance no pair is within, bit for bit."""
    from rl_collision_avoidance_b200.orca import noncoop_host, orca_host
    cfg, pose, goal, meta = _states(scenario, worlds, ticks, seed)
    R, N = cfg.robots_per_world, pose.shape[0]
    nd = 1e-3
    for w in range(worlds):
        p = pose[w * R:(w + 1) * R, 0:2].astype(np.float64)
        d = np.hypot(*(p[:, None] - p[None]).transpose(2, 0, 1)) + np.eye(R) * 1e9
        assert d.min() >= nd, (w, d.min())
    want, _, status = orca_host(cfg, pose, goal, meta, neighbour_dist=nd, heading_gain=2.0)
    assert not status.any()
    got = noncoop_host(cfg, pose, goal, meta, np.ones(N, np.uint8), _sentinel(np.random.default_rng(0), N))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert (got[:, 0] > 0).any()


@pytest.mark.parametrize('scenario,worlds,ticks,seed', STATES)
def test_slower_driver_matches_float64_and_keeps_unmasked_rows(built, scenario, worlds, ticks, seed):
    """speed < v_max on a random mask: masked rows agree with pref + tracker restated in float64 to 1e-5, with agents
    on every tracker branch (still on the goal, turning in place, driving); unmasked rows keep their bits."""
    from rl_collision_avoidance_b200.orca import noncoop_host
    cfg, pose, goal, meta = _states(scenario, worlds, ticks, seed)
    N = pose.shape[0]
    rng = np.random.default_rng(seed)
    goal[::5, 0:2] = pose[::5, 0:2]                                  # on the goal: v_pref = 0
    th = pose[1::5, 2].astype(np.float64)
    # behind and to one side: turn in place
    goal[1::5, 0:2] = pose[1::5, 0:2] + np.stack((-2.0 * np.cos(th) - np.sin(th), -2.0 * np.sin(th) + np.cos(th)), 1)
    mask = (rng.random(N) < 0.7).astype(np.uint8)
    mask[::5] = mask[1::5] = 1
    act0 = _sentinel(rng, N)
    speed, gain = 0.6, 1.5
    got = noncoop_host(cfg, pose, goal, meta, mask, act0, speed=speed, heading_gain=gain)
    keep = mask == 0
    assert keep.any() and np.array_equal(got[keep].view(np.uint32), act0[keep].view(np.uint32))
    pos, th, _ = orca_ref.agent_state(pose, goal, meta)
    branches = {'still': 0, 'turn': 0, 'drive': 0}
    for a in np.flatnonzero(mask):
        v = orca_ref.preferred(pos[a], goal[a, 0:2], speed, float(cfg.dt))
        want = orca_ref.track(th[a], v, speed, cfg.w_min, cfg.w_max, gain)
        assert np.abs(got[a] - want).max() <= 1e-5, (a, got[a], want)
        branches['still' if np.hypot(*v) <= 1e-6 else 'turn' if want[0] == 0 else 'drive'] += 1
        assert got[a, 0] <= np.float32(speed)
    assert all(branches.values()), branches


def test_bad_arguments_raise(built):
    from rl_collision_avoidance_b200.orca import noncoop_host
    cfg, pose, goal, meta = _states('stage1', 1, 1, 0)
    N = pose.shape[0]
    mask, act = np.ones(N, np.uint8), np.zeros((N, 2), np.float32)
    for speed in (0.0, -0.5, 1.0001, math.nan, math.inf):
        with pytest.raises(_lib.RlcaError):
            noncoop_host(cfg, pose, goal, meta, mask, act, speed=speed)
    for gain in (0.0, -1.0, math.nan, math.inf):
        with pytest.raises(_lib.RlcaError):
            noncoop_host(cfg, pose, goal, meta, mask, act, heading_gain=gain)
    with pytest.raises(ValueError):
        noncoop_host(cfg, pose, goal, meta, mask[:-1], act)
    lib = _lib.load()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    args = [vp(pose), vp(goal), vp(meta), vp(mask), 1.0, 2.0, vp(act)]
    for i in (0, 1, 2, 3, 6):
        bad = list(args)
        bad[i] = None
        assert lib.rlca_noncoop_action_host(C.byref(cfg), *bad) == 1, i
    assert lib.rlca_noncoop_action_host(None, *args) == 1
    # the device entry checks its arguments before it launches anything
    st = _lib.EnvState(vp(pose), vp(goal), None, vp(meta))
    assert lib.rlca_noncoop_action(C.byref(cfg), None, vp(mask), 1.0, 2.0, vp(act), None) == 1
    assert lib.rlca_noncoop_action(C.byref(cfg), C.byref(st), None, 1.0, 2.0, vp(act), None) == 1
    assert lib.rlca_noncoop_action(C.byref(cfg), C.byref(st), vp(mask), 1.0, 2.0, None, None) == 1
    assert lib.rlca_noncoop_action(C.byref(cfg), C.byref(st), vp(mask), 1.5, 2.0, vp(act), None) == 1
    assert lib.rlca_noncoop_action(C.byref(cfg), C.byref(st), vp(mask), 1.0, 0.0, vp(act), None) == 1


# ---------------------------------------------------------------------------------------------- split reduction
DT, GOAL_R, VMAX = 0.1, 0.5, 1.0


def _cfg(worlds, robots):
    return fill_config(_lib.EnvConfig(), make_scenario('stage1', robots_per_world=robots), num_worlds=worlds,
                       beams=512)


def _records(rng, W, R, E):
    N = W * R
    rec = np.zeros((N, E, 4), np.float32)
    rec[..., 0] = rng.choice([1, 1, 1, 2, 3], size=(N, E))
    rec[..., 1] = rng.integers(1, 152, size=(N, E))
    rec[..., 3] = rng.uniform(0.0, 12.0, size=(N, E))
    rec[..., 2] = rec[..., 3] * rng.uniform(0.9, 2.0, size=(N, E))
    count = rng.integers(0, E + 2, size=N).astype(np.int32)
    open_ = rng.integers(0, 2, size=N).astype(np.int32)
    return rec, count, open_


def _numpy_subset(rec, count, open_, agents, E):
    """The §9c definitions in float64 over `agents` in order (agent, then record)."""
    dt = float(np.float32(DT))
    s = np.zeros(NPARTIALS)
    for a in agents:
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
    return s


def test_split_with_zero_mask_is_the_unsplit_reduction(built):
    from rl_collision_avoidance_b200.evaluation import reduce_host, reduce_split_host
    W, R, E = 5, 24, 3
    rec, count, open_ = _records(np.random.default_rng(7), W, R, E)
    cfg = _cfg(W, R)
    split = reduce_split_host(cfg, rec, count, open_, np.zeros(W * R, np.uint8))
    assert split.shape == (W, 2, NPARTIALS)
    assert np.array_equal(split[:, 0].view(np.uint64), reduce_host(cfg, rec, count, open_).view(np.uint64))
    assert not split[:, 1].any()


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_split_rows_against_numpy(built, seed):
    """Random masks and records: each row is the numpy reduction of its subset, bit for bit; the counts of the two rows
    add up to the unsplit counts exactly; any world range gives the same rows."""
    from rl_collision_avoidance_b200.evaluation import reduce_host, reduce_split_host
    rng = np.random.default_rng(100 + seed)
    W, R, E = 6, 24, 3
    rec, count, open_ = _records(rng, W, R, E)
    mask = (rng.random(W * R) < 0.3).astype(np.uint8) * rng.integers(1, 256, W * R).astype(np.uint8)
    cfg = _cfg(W, R)
    split = reduce_split_host(cfg, rec, count, open_, mask)
    for w in range(W):
        agents = np.arange(w * R, (w + 1) * R)
        for row, sel in ((0, mask[agents] == 0), (1, mask[agents] != 0)):
            ref = _numpy_subset(rec, count, open_, agents[sel], E)
            assert np.array_equal(split[w, row].view(np.uint64), ref.view(np.uint64)), (w, row)
    full = reduce_host(cfg, rec, count, open_)
    assert np.array_equal(split[:, 0, :4] + split[:, 1, :4], full[:, :4])
    assert np.array_equal(reduce_split_host(cfg, rec, count, open_, mask, 2, 3), split[2:5])
    assert np.array_equal(reduce_split_host(cfg, rec, count, open_, mask, 5, 1), split[5:6])


def test_split_rejects_bad_arguments(built):
    from rl_collision_avoidance_b200.evaluation import reduce_split_host
    cfg = _cfg(2, 24)
    z = np.zeros((48, 1, 4), np.float32)
    zi = np.zeros(48, np.int32)
    m = np.zeros(48, np.uint8)
    for wb, wc in ((-1, 1), (0, 3), (2, 1), (1, 0)):
        with pytest.raises(_lib.RlcaError):
            reduce_split_host(cfg, z, zi, zi, m, wb, wc)
    with pytest.raises(ValueError):
        reduce_split_host(cfg, z, zi, zi, m[:-1])
    lib = _lib.load()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    out = np.zeros((2, 2, NPARTIALS))
    assert lib.rlca_eval_reduce_split_host(C.byref(cfg), vp(z), vp(zi), vp(zi), None, 1, 0, 2, vp(out)) == 1
    ev = _lib.EvalState(None, vp(zi), vp(zi), vp(zi), vp(z), 1)
    assert lib.rlca_eval_reduce_split(C.byref(cfg), C.byref(ev), None, 0, 2, vp(out), None) == 1


# ---------------------------------------------------------------------------------------------- helpers and CLI
def test_non_cooperative_mask():
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    m = non_cooperative_mask(24, 2, 5)
    assert m.dtype == np.uint8 and m.shape == (48,)
    assert list(np.flatnonzero(m)) == [0, 4, 9, 14, 19, 24, 28, 33, 38, 43]
    assert list(np.flatnonzero(non_cooperative_mask(50, 1, 1))) == [0]
    assert non_cooperative_mask(50, 3, 50).all()
    assert list(np.flatnonzero(non_cooperative_mask(2, 1, 2))) == [0, 1]
    for k in (0, -1, 25):
        with pytest.raises(ValueError):
            non_cooperative_mask(24, 2, k)


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'stage1', '--non-cooperative', '0'], '--non-cooperative must be in 1..24'),
    (['--scenario', 'stage1', '--non-cooperative', '25'], '--non-cooperative must be in 1..24'),
    (['--scenario', 'stage2', '--non-cooperative', '-3'], '--non-cooperative must be in 1..'),
    (['--scenario', 'circle', '--circle-robots', '8', '--non-cooperative', '9'], '--non-cooperative must be in 1..8'),
    (['--scenario', 'stage1', '--non-cooperative', '2', '--non-cooperative-speed', '0'],
     '--non-cooperative-speed must be in (0, 1]'),
    (['--scenario', 'stage1', '--non-cooperative', '2', '--non-cooperative-speed', '1.5'],
     '--non-cooperative-speed must be in (0, 1]'),
    (['--scenario', 'stage1', '--non-cooperative', '2', '--non-cooperative-speed', 'nan'],
     '--non-cooperative-speed must be in (0, 1]'),
    (['--scenario', 'stage1', '--non-cooperative-speed', '0.5'], '--non-cooperative-speed applies with'),
])
@pytest.mark.parametrize('who', [['--policy', os.path.join(CKPT, 'stage2.pth')], ['--baseline', 'nh-orca']])
def test_evaluate_cli_rejects_bad_non_cooperative(capsys, argv, message, who):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(argv + who)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


@pytest.mark.parametrize('obj, kernel', [('rlca_orca.o', 'rlca_noncoop_kernel'),
                                         ('rlca_eval.o', 'eval_reduce_split_kernel')])
def test_new_kernels_do_not_spill(built, obj, kernel):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', obj)], check=True,
                         capture_output=True, text=True).stdout
    m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % kernel, out)
    assert m, out
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
    assert int(m.group(1)) <= 128, m.group(0)
