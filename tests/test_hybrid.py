"""The hybrid controller without a GPU (DESIGN.md §9j): rlca_hybrid_action_host against a numpy restatement on oracle
states of every scenario, the boundaries of both strict tests, the disabled setting, the counters, every rejected
argument (ABI, Hybrid, evaluate.py) and the register budget of the kernel."""
import ctypes as C
import math
import os
import re
import subprocess
import types

import numpy as np
import pytest

from helpers import make_pair, random_actions
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.evaluation import AUTO_RESET
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario, random_layout_host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
F = np.float32


def _states(scenario, worlds, ticks, seed, robots=None):
    """EnvConfig, (N, 3, beams) scan stack of the last three ticks (frame 2 newest) and (pose, goal, meta) of the CPU
    oracle after `ticks` random-action ticks; a random scenario is laid out first."""
    sc, _, orc = make_pair(scenario, num_worlds=worlds, gpu=False, seed=seed, auto_reset=AUTO_RESET[scenario],
                           robots_per_world=robots)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=worlds, beams=512, auto_reset=AUTO_RESET[scenario], seed=seed)
    orc.reset_world()
    orc.reset_pose()
    if sc.layout is not None:
        pose, goal, acc, status = random_layout_host(cfg, sc.layout, orc.pose, orc.goal, orc.acc)
        assert not status.any()
        orc.pose[...], orc.goal[...], orc.acc[...] = pose, goal, acc
        orc.observe()
    rng = np.random.default_rng(seed)
    frames = [orc.obs.copy()] * 3
    for _ in range(ticks):
        orc.step(random_actions(rng, orc.N))
        frames = frames[1:] + [orc.obs.copy()]
    return cfg, np.ascontiguousarray(np.stack(frames, 1)), orc.pose.copy(), orc.goal.copy(), orc.meta.copy()


STATES = [('stage1', 3, 12, 1, None), ('stage2', 2, 12, 2, None), ('circle', 1, 12, 3, None),
          ('random', 6, 12, 4, 8)]


def _distance(cfg, stack):
    """d per agent in metres, float32 as the library computes it."""
    return (stack[:, 2].min(1) + F(0.5)) * F(cfg.range_max)


def _sentinel(rng, n):
    act = rng.uniform(-5, 5, (n, 2)).astype(np.float32)
    act[::7, 0] = np.nan
    act[3::7, 1] = np.nan
    return act


def _restated(cfg, stack, pose, goal, meta, action, open_, counts, r_safe, r_risk, v_safe, gain):
    """The §9j definition in numpy; the driver's rows from noncoop_host with an all-ones mask."""
    from rl_collision_avoidance_b200.orca import noncoop_host
    d = _distance(cfg, stack)
    mode = np.where(d > F(r_safe), 1, np.where(d < F(r_risk), 2, 0)).astype(np.uint8)
    drv = noncoop_host(cfg, pose, goal, meta, np.ones(len(d), np.uint8), action, heading_gain=gain)
    act = action.copy()
    act[mode == 1] = drv[mode == 1]
    act[mode == 2, 0] = np.fmin(act[mode == 2, 0], F(v_safe))
    cnt = counts.copy()
    cnt[np.arange(len(d)), mode] += (open_ != 0).astype(np.int32)
    return act, mode, cnt


def _bits(a):
    return np.asarray(a).view(np.uint32)


@pytest.mark.parametrize('scenario,worlds,ticks,seed,robots', STATES)
def test_host_equals_numpy_restatement(built, scenario, worlds, ticks, seed, robots):
    """Thresholds at the 1/3 and 2/3 quantiles of d (every mode occurs): action, mode and counts equal the restatement
    bit for bit.  Driver rows are the §9h driver's, policy rows keep a NaN-laced sentinel, safe rows are min(v, v_safe)
    and keep w; the defaults and another gain and cap agree too."""
    from rl_collision_avoidance_b200.orca import HYBRID_DEFAULTS, hybrid_host, noncoop_host
    cfg, stack, pose, goal, meta = _states(scenario, worlds, ticks, seed, robots)
    N = pose.shape[0]
    rng = np.random.default_rng(seed)
    d = _distance(cfg, stack)
    lo, hi = (float(np.quantile(d, q, method='lower')) for q in (1 / 3, 2 / 3))
    open_ = (rng.random(N) < 0.8).astype(np.int32) * rng.integers(1, 5, N).astype(np.int32)
    counts0 = rng.integers(0, 1000, (N, 3)).astype(np.int32)
    act0 = _sentinel(rng, N)
    for r_safe, r_risk, v_safe, gain in ((hi, lo, 0.5, 2.0), (hi, lo, 0.3, 1.5),
                                         tuple(HYBRID_DEFAULTS[k] for k in ('r_safe', 'r_risk', 'v_safe',
                                                                             'heading_gain'))):
        got = hybrid_host(cfg, stack, pose, goal, meta, act0, open_, counts0, r_safe=r_safe, r_risk=r_risk,
                          v_safe=v_safe, heading_gain=gain)
        want = _restated(cfg, stack, pose, goal, meta, act0, open_, counts0, r_safe, r_risk, v_safe, gain)
        assert np.array_equal(_bits(got[0]), _bits(want[0]))
        assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
        mode = got[1]
        if r_safe == hi:
            assert all((mode == k).any() for k in range(3)), np.bincount(mode)
        drv = noncoop_host(cfg, pose, goal, meta, np.ones(N, np.uint8), act0, heading_gain=gain)
        assert np.array_equal(_bits(got[0][mode == 1]), _bits(drv[mode == 1]))
        assert np.array_equal(_bits(got[0][mode == 0]), _bits(act0[mode == 0]))
        safe = mode == 2
        assert np.array_equal(_bits(got[0][safe, 1]), _bits(act0[safe, 1]))
        assert np.array_equal(_bits(got[0][safe, 0]), _bits(np.fmin(act0[safe, 0], F(v_safe))))
        assert (got[0][safe, 0] <= F(v_safe)).all()


def _hand_stack(cfg, n, m):
    """(n, 3, beams) stacks whose frame 2 has minimum m[a] at one beam and 0.5 (a miss) elsewhere; frames 0 and 1 are
    all hits at -0.5, which the hybrid must not read."""
    beams = cfg.beams
    s = np.full((n, 3, beams), -0.5, np.float32)
    s[:, 2] = 0.5
    s[np.arange(n), 2, (np.arange(n) * 37) % beams] = m
    return s


def test_boundaries_are_policy_mode(built):
    """d exactly at r_safe and exactly at r_risk is mode 0: both tests are strict."""
    from rl_collision_avoidance_b200.orca import hybrid_host
    cfg, _, pose, goal, meta = _states('stage1', 1, 2, 0)
    N = pose.shape[0]
    rng = np.random.default_rng(5)
    m = rng.uniform(-0.45, 0.45, N).astype(np.float32)
    d = (m + F(0.5)) * F(cfg.range_max)
    stack = _hand_stack(cfg, N, m)
    act0 = _sentinel(rng, N)
    for a in range(N):
        da = float(d[a])
        for r_safe, r_risk in ((da, 0.0), (da, da), (float(cfg.range_max), da)):
            act, mode, _ = hybrid_host(cfg, stack[a:a + 1].repeat(N, 0), pose, goal, meta, act0, r_safe=r_safe,
                                       r_risk=r_risk)
            assert not mode.any(), (a, r_safe, r_risk)
            assert np.array_equal(_bits(act), _bits(act0))
        # one ulp either side leaves the boundary
        below, above = float(np.nextafter(d[a], F(-1))), float(np.nextafter(d[a], F(10)))
        assert hybrid_host(cfg, stack[a:a + 1].repeat(N, 0), pose, goal, meta, act0, r_safe=below,
                           r_risk=0.0)[1].all()
        assert (hybrid_host(cfg, stack[a:a + 1].repeat(N, 0), pose, goal, meta, act0, r_safe=above,
                            r_risk=above)[1] == 2).all()


@pytest.mark.parametrize('scenario,worlds,ticks,seed,robots', STATES)
def test_disabled_leaves_every_action(built, scenario, worlds, ticks, seed, robots):
    """r_risk = 0 and r_safe = range_max: every row is mode 0 and keeps its bits; a stack of misses stays mode 0."""
    from rl_collision_avoidance_b200.orca import hybrid_host
    cfg, stack, pose, goal, meta = _states(scenario, worlds, ticks, seed, robots)
    N = pose.shape[0]
    act0 = _sentinel(np.random.default_rng(seed), N)
    for s in (stack, _hand_stack(cfg, N, np.full(N, 0.5, np.float32)), _hand_stack(cfg, N, np.full(N, -0.5, F))):
        act, mode, cnt = hybrid_host(cfg, s, pose, goal, meta, act0, np.ones(N, np.int32), r_safe=cfg.range_max,
                                     r_risk=0.0)
        assert not mode.any()
        assert np.array_equal(_bits(act), _bits(act0))
        assert (cnt[:, 0] == 1).all() and not cnt[:, 1:].any()


def test_counts_move_only_where_open(built):
    from rl_collision_avoidance_b200.orca import hybrid_host
    cfg, stack, pose, goal, meta = _states('stage2', 2, 6, 9)
    N = pose.shape[0]
    rng = np.random.default_rng(9)
    d = _distance(cfg, stack)
    lo, hi = (float(np.quantile(d, q, method='lower')) for q in (1 / 3, 2 / 3))
    counts = rng.integers(0, 50, (N, 3)).astype(np.int32)
    open_ = (rng.random(N) < 0.5).astype(np.int32)
    act0 = _sentinel(rng, N)
    total = counts.copy()
    for t in range(4):
        act, mode, total = hybrid_host(cfg, stack, pose, goal, meta, act0, open_, total, r_safe=hi, r_risk=lo)
    assert np.array_equal(total[open_ == 0], counts[open_ == 0])
    want = counts + 4 * np.eye(3, dtype=np.int32)[mode] * open_[:, None]
    assert np.array_equal(total, want)
    # without open nothing is counted, and the counters passed in come back unchanged
    _, mode2, same = hybrid_host(cfg, stack, pose, goal, meta, act0, None, counts, r_safe=hi, r_risk=lo)
    assert np.array_equal(same, counts) and np.array_equal(mode2, mode)


BAD = [dict(r_safe=2.0, r_risk=2.5), dict(r_risk=-0.1), dict(r_safe=6.5, r_risk=0.5), dict(r_safe=math.inf),
       dict(r_safe=math.nan), dict(r_risk=math.nan), dict(r_risk=-math.inf), dict(v_safe=0.0), dict(v_safe=-0.5),
       dict(v_safe=1.0001), dict(v_safe=math.nan), dict(v_safe=math.inf), dict(heading_gain=0.0),
       dict(heading_gain=-1.0), dict(heading_gain=math.nan), dict(heading_gain=math.inf)]


def _params(**kw):
    from rl_collision_avoidance_b200.orca import HYBRID_DEFAULTS
    p = dict(HYBRID_DEFAULTS)
    p.update(kw)
    return p


@pytest.mark.parametrize('bad', BAD)
def test_bad_parameters_are_rejected_everywhere(built, bad):
    """Both ABI entries return RLCA_ERR_INVALID (the device entry before it launches anything) and Hybrid raises
    ValueError before it touches a device."""
    from rl_collision_avoidance_b200.orca import Hybrid
    cfg, stack, pose, goal, meta = _states('stage1', 1, 1, 0)
    N = pose.shape[0]
    lib = _lib.load()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    act, mode, opn, cnt = np.zeros((N, 2), F), np.zeros(N, np.uint8), np.ones(N, np.int32), np.zeros((N, 3), np.int32)
    prm = _lib.HybridParams(**_params(**bad))
    assert lib.rlca_hybrid_action_host(C.byref(cfg), C.byref(prm), vp(stack), vp(pose), vp(goal), vp(meta), vp(opn),
                                       vp(act), vp(mode), vp(cnt)) == 1
    st = _lib.EnvState(vp(pose), vp(goal), None, vp(meta))
    assert lib.rlca_hybrid_action(C.byref(cfg), C.byref(prm), C.byref(st), vp(stack), vp(opn), vp(act), vp(mode),
                                  vp(cnt), None) == 1
    env = types.SimpleNamespace(cfg=cfg, N=N, device='no-device')
    with pytest.raises(ValueError):
        Hybrid(env, **_params(**bad))


def test_bad_buffers_are_rejected(built):
    from rl_collision_avoidance_b200.orca import hybrid_host
    cfg, stack, pose, goal, meta = _states('stage1', 1, 1, 0)
    N = pose.shape[0]
    lib = _lib.load()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    act, mode, opn, cnt = np.zeros((N, 2), F), np.zeros(N, np.uint8), np.ones(N, np.int32), np.zeros((N, 3), np.int32)
    prm = _lib.HybridParams(**_params())
    args = [vp(stack), vp(pose), vp(goal), vp(meta), vp(opn), vp(act), vp(mode), vp(cnt)]
    assert lib.rlca_hybrid_action_host(C.byref(cfg), C.byref(prm), *args) == 0
    for i in (0, 1, 2, 3, 4, 5, 6, 7):
        bad = list(args)
        bad[i] = None
        assert lib.rlca_hybrid_action_host(C.byref(cfg), C.byref(prm), *bad) == 1, i
    assert lib.rlca_hybrid_action_host(C.byref(cfg), C.byref(prm), *args[:4], None, *args[5:7], None) == 0
    assert lib.rlca_hybrid_action_host(None, C.byref(prm), *args) == 1
    assert lib.rlca_hybrid_action_host(C.byref(cfg), None, *args) == 1
    st = _lib.EnvState(vp(pose), vp(goal), None, vp(meta))
    dev = [vp(stack), vp(opn), vp(act), vp(mode), vp(cnt)]
    for i in range(5):
        bad = list(dev)
        bad[i] = None
        assert lib.rlca_hybrid_action(C.byref(cfg), C.byref(prm), C.byref(st), *bad, None) == 1, i
    assert lib.rlca_hybrid_action(C.byref(cfg), C.byref(prm), None, *dev, None) == 1
    assert lib.rlca_hybrid_action(C.byref(cfg), None, C.byref(st), *dev, None) == 1
    for k in ('pose_dev', 'goal_dev', 'meta_dev'):
        st2 = _lib.EnvState(vp(pose), vp(goal), None, vp(meta))
        setattr(st2, k, None)
        assert lib.rlca_hybrid_action(C.byref(cfg), C.byref(prm), C.byref(st2), *dev, None) == 1, k
    with pytest.raises(ValueError):
        hybrid_host(cfg, stack[:, :2], pose, goal, meta, act)
    with pytest.raises(ValueError):
        hybrid_host(cfg, stack, pose, goal, meta, act, opn[:-1])


def test_mode_shares():
    from rl_collision_avoidance_b200.orca import mode_shares
    s = mode_shares(np.array([[3, 1, 0], [5, 0, 1]], np.int64))
    assert s == {'policy': 0.8, 'driver': 0.1, 'safe': 0.1, 'agent_ticks': 10}
    z = mode_shares(np.zeros((2, 3), np.int64))
    assert z['agent_ticks'] == 0 and all(math.isnan(z[k]) for k in ('policy', 'driver', 'safe'))


POLICY = ['--policy', os.path.join(CKPT, 'stage2.pth')]


@pytest.mark.parametrize('argv, message', [
    (POLICY + ['--hybrid-r-safe', '3'], 'apply with --hybrid only'),
    (POLICY + ['--hybrid-r-risk', '0.5'], 'apply with --hybrid only'),
    (POLICY + ['--hybrid-v-safe', '0.3'], 'apply with --hybrid only'),
    (['--baseline', 'nh-orca', '--hybrid'], '--hybrid applies to --policy only'),
    (['--baseline', 'orca', '--hybrid', '--hybrid-r-safe', '3'], '--hybrid applies to --policy only'),
    (POLICY + ['--hybrid', '--hybrid-r-safe', '0.5'], 'need 0 <= r_risk <= r_safe <= range_max'),
    (POLICY + ['--hybrid', '--hybrid-r-safe', '6.5'], 'need 0 <= r_risk <= r_safe <= range_max'),
    (POLICY + ['--hybrid', '--hybrid-r-safe', 'inf'], 'need 0 <= r_risk <= r_safe <= range_max'),
    (POLICY + ['--hybrid', '--hybrid-r-risk', '-1'], 'need 0 <= r_risk <= r_safe <= range_max'),
    (POLICY + ['--hybrid', '--hybrid-r-risk', 'nan'], 'need 0 <= r_risk <= r_safe <= range_max'),
    (POLICY + ['--hybrid', '--hybrid-v-safe', '0'], 'v_safe must be in (0, 1]'),
    (POLICY + ['--hybrid', '--hybrid-v-safe', '1.5'], 'v_safe must be in (0, 1]'),
    (POLICY + ['--hybrid', '--hybrid-v-safe', 'nan'], 'v_safe must be in (0, 1]'),
])
@pytest.mark.parametrize('scenario', [['--scenario', 'stage1'], ['--scenario', 'random', '--random-robots', '8'],
                                      ['--scenario', 'circle', '--circle-robots', '8', '--non-cooperative', '2']])
def test_evaluate_cli_rejects_bad_hybrid(capsys, argv, message, scenario):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(scenario + argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_kernel_does_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_orca.o')], check=True,
                         capture_output=True, text=True).stdout
    m = re.search(r'Function \w*rlca_hybrid_kernel\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', out)
    assert m, out
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
    assert int(m.group(1)) <= 64, m.group(0)
