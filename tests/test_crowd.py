"""The social-force crowd without a GPU (DESIGN.md §9t): dev_expf against float64 exp, rlca_crowd_action_host against a
float64 restatement (tests/crowd_ref.py) on oracle states with and without the map, the rows it must not touch, its
degenerate cases, every argument check and command-line rule, the kernel's register budget, the trainers' filter of
masked rows, and the head-on pair that the straight driver crashes."""
import ctypes as C
import math
import os
import re
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import crowd_ref
from helpers import make_pair, random_actions
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.evaluation import AUTO_RESET
from rl_collision_avoidance_b200.scenarios import fill_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
TOL = 1e-5
EXPF_ULP = 1            # dev_expf is a faithful rounding: the largest error over the sweep below is 0.99 ulp


def _ulp_error(got, x):
    want = np.exp(x.astype(np.float64))
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    return np.abs(got.astype(np.float64) - want) / ulp


def _expf(x):
    lib = _lib.load()
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(x)
    _lib.check(lib.rlca_crowd_expf_host(x.ctypes.data_as(C.c_void_p), x.size, out.ctypes.data_as(C.c_void_p)))
    return out


def test_dev_expf_against_float64(built):
    """Within EXPF_ULP ulp of float64 exp over every normal result (dense over [-20, 10], where the kernel's arguments
    lie with the defaults: agents [(2r - nd) / range, 2r / range) = [-4.6, 1.4), walls [-6.5, 3.5)), exact at 0, inf
    above ln(FLT_MAX), 0 below ln(FLT_MIN)."""
    rng = np.random.default_rng(0)
    x = np.concatenate((np.linspace(-20, 10, 400001, dtype=np.float32), rng.uniform(-87.3, 88.7, 200000)
                        .astype(np.float32), np.float32([-87.33, 88.72, 1e-8, -1e-8, 0.5, -0.5])))
    got = _expf(x)
    err = _ulp_error(got, x)
    assert err.max() <= EXPF_ULP, (err.max(), x[np.argmax(err)])
    assert _expf(np.float32([0.0]))[0] == 1.0
    edge = _expf(np.float32([89.0, 1e30, -88.0, -1e30, np.inf, -np.inf, np.nan]))
    assert np.isinf(edge[0]) and np.isinf(edge[1]) and edge[2] == 0 and edge[3] == 0
    assert np.isinf(edge[4]) and edge[5] == 0 and np.isnan(edge[6])


# ---------------------------------------------------------------------------------------------- host twin
def _states(scenario, worlds, ticks, seed):
    sc, _, orc = make_pair(scenario, num_worlds=worlds, gpu=False, seed=seed, auto_reset=AUTO_RESET[scenario])
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(seed)
    for _ in range(ticks):
        orc.step(random_actions(rng, orc.N))
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=worlds, beams=512, auto_reset=AUTO_RESET[scenario], seed=seed)
    return sc, cfg, orc.pose.copy(), orc.goal.copy(), orc.meta.copy()


def _inject(pose, goal, R):
    """World 0 gets the corner cases; returns the agents that must be masked: 0 on its goal, 1 and 2 coincident, 3 and
    4 in contact (0.4 m apart, below 2 radius), 5 exactly neighbour_dist = 3 m from 6."""
    pose[0, 0:2] = (2.0, 2.5)
    goal[0, 0:2] = pose[0, 0:2]
    pose[2, 0:2] = pose[1, 0:2]
    pose[4, 0:2] = pose[3, 0:2] + np.float32([0.25, 0.3125])
    pose[5, 0:2] = (-1.0, 6.0)
    pose[6, 0:2] = (2.0, 6.0)
    return [0, 1, 2, 3, 4, 5, 6]


def _sentinel(rng, n):
    act = rng.uniform(-5, 5, (n, 2)).astype(np.float32)
    act[::7, 0] = np.nan
    return act


STATES = [('stage1', 3, 12, 1), ('stage2', 2, 12, 2), ('circle', 1, 12, 3)]


@pytest.mark.parametrize('scenario,worlds,ticks,seed', STATES)
@pytest.mark.parametrize('see_robots', [True, False])
@pytest.mark.parametrize('with_map', [False, True])
def test_host_twin_matches_float64(built, scenario, worlds, ticks, seed, see_robots, with_map):
    """Masked rows agree with the float64 restatement to 1e-5, on every tracker branch and with the corner cases of
    _inject; agents with a distance within 1e-4 of a cut-off (but not on it) are left out, as float32 rounding may
    decide those either way.  Unmasked rows keep their bits."""
    from rl_collision_avoidance_b200.crowd import CrowdParams, crowd_host
    from rl_collision_avoidance_b200.orca import ObstacleSet
    if with_map and scenario != 'stage2':
        pytest.skip('the map is stage 2\'s obstacle set')
    sc, cfg, pose, goal, meta = _states(scenario, worlds, ticks, seed)
    R, N = cfg.robots_per_world, pose.shape[0]
    rng = np.random.default_rng(seed)
    special = _inject(pose, goal, R)
    mask = (rng.random(N) < 0.5).astype(np.uint8) * rng.integers(1, 256, N).astype(np.uint8)
    mask[special] = 1
    params = CrowdParams(speed=0.8, see_robots=see_robots)
    obs, segs = None, None
    if with_map:
        obs = ObstacleSet(cfg, sc.map.cells, params.wall_dist)
        segs = obs.segments()[0]
    act0 = _sentinel(rng, N)
    got = crowd_host(cfg, pose, goal, meta, mask, act0, params, obstacles=obs)
    keep = mask == 0
    assert np.array_equal(got[keep].view(np.uint32), act0[keep].view(np.uint32))
    checked, walls, branches = 0, 0, {'still': 0, 'turn': 0, 'drive': 0}
    for a in np.flatnonzero(mask):
        d = crowd_ref.distances(cfg, pose, a, segs)
        near = np.concatenate((d[:R - 1] - params.neighbour_dist, d[R - 1:] - params.wall_dist))
        if ((np.abs(near) < 1e-4) & (near != 0)).any():
            continue
        want = crowd_ref.crowd_action(cfg, pose, goal, meta, mask, a, params, segs)
        assert np.abs(got[a] - want).max() <= TOL, (a, got[a], want)
        checked += 1
        walls += bool(segs is not None and crowd_ref.wall_terms(pose[a, 0:2].astype(np.float64), segs, 1.0))
        branches['still' if not got[a].any() else 'turn' if got[a, 0] == 0 else 'drive'] += 1
    assert checked >= 0.9 * np.count_nonzero(mask), checked
    assert branches['drive'] and branches['turn'] + branches['still'], branches
    if with_map:
        assert walls > 0


def test_corner_cases(built):
    """On its goal with no neighbour the agent stands still; a coincident pair adds no force; a neighbour exactly at
    neighbour_dist adds none, one just inside does."""
    from rl_collision_avoidance_b200.crowd import CrowdParams, crowd_host
    _, cfg, pose, goal, meta = _states('circle', 1, 0, 4)
    R = cfg.robots_per_world
    pose[:, 0:2] = np.stack((np.arange(R) * 20.0, np.full(R, 40.0)), 1)     # nobody within 3 m of anyone
    meta[:, 2] = 1                                                          # standing: v = 0
    mask = np.zeros(R, np.uint8)
    mask[:4] = 1
    p = CrowdParams()
    goal[0, 0:2] = pose[0, 0:2]
    act = crowd_host(cfg, pose, goal, meta, mask, np.zeros((R, 2), np.float32), p)
    assert not act[0].any()
    alone = act[1].copy()
    pose[2, 0:2] = pose[1, 0:2]                                             # coincident with 1
    assert np.array_equal(crowd_host(cfg, pose, goal, meta, mask, np.zeros((R, 2), np.float32), p)[1], alone)
    pose[2, 0:2] = pose[1, 0:2] + np.float32([0.0, 3.0])                    # exactly at the cut-off
    assert np.array_equal(crowd_host(cfg, pose, goal, meta, mask, np.zeros((R, 2), np.float32), p)[1], alone)
    pose[2, 0:2] = pose[1, 0:2] + np.float32([0.0, 2.5])
    assert not np.array_equal(crowd_host(cfg, pose, goal, meta, mask, np.zeros((R, 2), np.float32), p)[1], alone)


def test_all_free_grid_is_map_blind(built):
    from rl_collision_avoidance_b200.crowd import CrowdParams, crowd_host
    from rl_collision_avoidance_b200.orca import ObstacleSet
    sc, cfg, pose, goal, meta = _states('stage2', 2, 10, 5)
    N = pose.shape[0]
    mask = np.ones(N, np.uint8)
    free = ObstacleSet(cfg, np.zeros_like(sc.map.cells), 1.0)
    act0 = _sentinel(np.random.default_rng(5), N)
    for see in (True, False):
        p = CrowdParams(see_robots=see)
        a = crowd_host(cfg, pose, goal, meta, mask, act0, p)
        b = crowd_host(cfg, pose, goal, meta, mask, act0, p, obstacles=free)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_invisible_robots_change_nothing(built):
    """see_robots False: moving the unmasked agents leaves every masked row's bits unchanged; with see_robots True the
    same move changes some."""
    from rl_collision_avoidance_b200.crowd import CrowdParams, crowd_host
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    sc, cfg, pose, goal, meta = _states('stage2', 3, 15, 6)
    N, R = pose.shape[0], cfg.robots_per_world
    mask = non_cooperative_mask(R, 3, 8)
    moved = pose.copy()
    rng = np.random.default_rng(6)
    moved[mask == 0, 0:2] += rng.normal(0, 0.5, (int((mask == 0).sum()), 2)).astype(np.float32)
    act0 = np.zeros((N, 2), np.float32)
    blind = CrowdParams(see_robots=False)
    a = crowd_host(cfg, pose, goal, meta, mask, act0, blind)
    b = crowd_host(cfg, moved, goal, meta, mask, act0, blind)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    c = crowd_host(cfg, pose, goal, meta, mask, act0, CrowdParams())
    d = crowd_host(cfg, moved, goal, meta, mask, act0, CrowdParams())
    assert not np.array_equal(c, d)


# ---------------------------------------------------------------------------------------------- argument checks
BAD = [('speed', 0.0), ('speed', -1.0), ('speed', math.nan), ('speed', math.inf)] + \
    [(k, v) for k in ('relax_time', 'range', 'wall_range', 'radius', 'neighbour_dist', 'heading_gain', 'wall_dist')
     for v in (0.0, -1.0, math.nan, math.inf)] + \
    [(k, v) for k in ('strength', 'wall_strength', 'side_bias') for v in (-0.1, math.nan, math.inf)] + \
    [('anisotropy', v) for v in (-0.01, 1.01, math.nan)]


@pytest.mark.parametrize('key,value', BAD)
def test_bad_parameters_raise(built, key, value):
    """CrowdParams refuses the value, and so does the library's own check of the same struct."""
    from rl_collision_avoidance_b200.crowd import CrowdParams
    with pytest.raises(ValueError):
        CrowdParams(**{key: value})
    _, cfg, pose, goal, meta = _states('stage1', 1, 0, 0)
    N = pose.shape[0]
    ps = CrowdParams().struct(cfg.v_max)
    setattr(ps, key, value)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    mask, act = np.ones(N, np.uint8), np.zeros((N, 2), np.float32)
    lib = _lib.load()
    assert lib.rlca_crowd_action_host(C.byref(cfg), C.byref(ps), None, vp(pose), vp(goal), vp(meta), vp(mask),
                                      vp(act)) == 1
    st = _lib.EnvState(vp(pose), vp(goal), None, vp(meta))
    assert lib.rlca_crowd_action(C.byref(cfg), C.byref(ps), C.byref(st), vp(mask), None, vp(act), None) == 1


def test_bad_buffers_and_ranges_raise(built):
    from rl_collision_avoidance_b200.crowd import CrowdParams, crowd_host
    from rl_collision_avoidance_b200.orca import ObstacleSet
    sc, cfg, pose, goal, meta = _states('stage2', 1, 0, 0)
    N = pose.shape[0]
    mask, act = np.ones(N, np.uint8), np.zeros((N, 2), np.float32)
    with pytest.raises(_lib.RlcaError):
        crowd_host(cfg, pose, goal, meta, mask, act, CrowdParams(speed=1.0001))
    short = ObstacleSet(cfg, sc.map.cells, 0.5)
    with pytest.raises(_lib.RlcaError):
        crowd_host(cfg, pose, goal, meta, mask, act, CrowdParams(), obstacles=short)
    crowd_host(cfg, pose, goal, meta, mask, act, CrowdParams(wall_dist=0.5), obstacles=short)
    with pytest.raises(ValueError):
        crowd_host(cfg, pose, goal, meta, mask[:-1], act)
    lib = _lib.load()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    ps = CrowdParams().struct(cfg.v_max)
    args = [vp(pose), vp(goal), vp(meta), vp(mask), vp(act)]
    for i in range(len(args)):
        bad = list(args)
        bad[i] = None
        assert lib.rlca_crowd_action_host(C.byref(cfg), C.byref(ps), None, *bad) == 1, i
    assert lib.rlca_crowd_action_host(None, C.byref(ps), None, *args) == 1
    assert lib.rlca_crowd_action_host(C.byref(cfg), None, None, *args) == 1
    st = _lib.EnvState(vp(pose), vp(goal), None, vp(meta))
    assert lib.rlca_crowd_action(C.byref(cfg), C.byref(ps), None, vp(mask), None, vp(act), None) == 1
    assert lib.rlca_crowd_action(C.byref(cfg), C.byref(ps), C.byref(st), None, None, vp(act), None) == 1
    assert lib.rlca_crowd_action(C.byref(cfg), C.byref(ps), C.byref(st), vp(mask), None, None, None) == 1
    assert lib.rlca_crowd_action(C.byref(cfg), C.byref(ps), C.byref(st), vp(mask), short.handle, vp(act), None) == 1


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'stage1', '--crowd', '2', '--non-cooperative', '2'], 'cannot be combined'),
    (['--scenario', 'stage1', '--crowd', '0'], '--crowd must be in 1..24'),
    (['--scenario', 'stage1', '--crowd', '25'], '--crowd must be in 1..24'),
    (['--scenario', 'circle', '--circle-robots', '8', '--crowd', '9'], '--crowd must be in 1..8'),
    (['--scenario', 'stage1', '--crowd-speed', '0.5'], '--crowd-speed applies with --crowd only'),
    (['--scenario', 'stage1', '--crowd-map'], '--crowd-map applies with --crowd only'),
    (['--scenario', 'stage1', '--crowd-ignores-robots'], '--crowd-ignores-robots applies with --crowd only'),
    (['--scenario', 'stage1', '--crowd-strength', '1'], '--crowd-strength applies with --crowd only'),
    (['--scenario', 'stage1', '--crowd', '2', '--crowd-speed', '1.5'], '--crowd-speed must be in (0, 1]'),
    (['--scenario', 'stage1', '--crowd', '2', '--crowd-speed', '0'], '--crowd-speed must be in (0, 1]'),
    (['--scenario', 'stage1', '--crowd', '2', '--crowd-strength', '-1'], 'strength must be finite and >= 0'),
    (['--scenario', 'stage1', '--crowd', '2', '--crowd-range', '0'], 'range must be finite and > 0'),
    (['--scenario', 'stage1', '--crowd', '2', '--crowd-side-bias', 'nan'], 'side_bias must be finite and >= 0'),
])
@pytest.mark.parametrize('who', [['--policy', os.path.join(CKPT, 'stage2.pth')], ['--baseline', 'nh-orca']])
def test_evaluate_cli_rejects_bad_crowd(capsys, argv, message, who):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(argv + who)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


@pytest.mark.parametrize('argv, message', [
    (['--crowd', '2', '--non-cooperative', '2'], 'cannot be combined'),
    (['--non-cooperative-speed', '0.5'], '--non-cooperative-speed applies with --non-cooperative only'),
    (['--non-cooperative', '0'], '--non-cooperative must be >= 1'),
    (['--non-cooperative', '2', '--non-cooperative-speed', '2'], '--non-cooperative-speed must be in (0, 1]'),
    (['--crowd', '0'], '--crowd must be in 1..'),
    (['--crowd-range', '0.4'], '--crowd-range applies with --crowd only'),
    (['--crowd', '2', '--crowd-range', '-1'], 'range must be finite and > 0'),
])
def test_trainer_cli_rejects_bad_masked_flags(capsys, argv, message):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(stage=2, argv=argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_kernel_does_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_orca.o')], check=True,
                         capture_output=True, text=True).stdout
    found = re.findall(r'Function \w*rlca_crowd_kernel\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', out)
    assert len(found) == 2, out
    for reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0 and int(reg) <= 64, (reg, stack, local)


# ---------------------------------------------------------------------------------------------- trainer filter
@pytest.mark.parametrize('seed', range(4))
def test_trainer_filter_is_reference_filter_and_masked_rows(seed):
    from rl_collision_avoidance_b200.model.utils import get_filter_index
    from rl_collision_avoidance_b200.trainer import masked_filter_index, masked_rows
    rng = np.random.default_rng(seed)
    H, N = int(rng.integers(1, 40)), int(rng.integers(1, 90))
    dones = rng.random((H, N)) < rng.uniform(0.05, 0.9)
    col = rng.random(N) < 0.3
    got = masked_filter_index(dones, col)
    want = set(int(i) for i in get_filter_index(dones)) | {t * N + i for t in range(H) for i in np.flatnonzero(col)}
    assert got == sorted(want)
    assert masked_rows(H, col) == sorted(t * N + i for t in range(H) for i in np.flatnonzero(col))
    assert masked_filter_index(dones, np.zeros(N, bool)) == sorted(set(int(i) for i in get_filter_index(dones)))


def _fake_comp(R, W):
    cfg = SimpleNamespace(robots_per_world=R, num_worlds=W, v_max=1.0)
    return SimpleNamespace(env=SimpleNamespace(cfg=cfg, N=R * W, device='cpu'), masked=None)


def test_masked_agents_per_component():
    """Each component gets non_cooperative_mask(R_c, W_c, k); k > R_c and both kinds at once are ValueErrors."""
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    from rl_collision_avoidance_b200.trainer import masked_agents
    comps = [_fake_comp(44, 2), _fake_comp(16, 3)]
    col = masked_agents(comps, non_cooperative=(3, 0.5))
    assert np.array_equal(col, np.concatenate((non_cooperative_mask(44, 2, 3), non_cooperative_mask(16, 3, 3))) != 0)
    assert comps[0].masked.speed == 0.5 and comps[1].masked.mask.sum() == 9
    assert masked_agents([_fake_comp(8, 1)]) is None
    with pytest.raises(ValueError):
        masked_agents([_fake_comp(44, 1), _fake_comp(16, 1)], non_cooperative=(17, None))
    with pytest.raises(ValueError):
        masked_agents([_fake_comp(8, 1)], non_cooperative=(1, None), crowd=(1, None, False))


# ---------------------------------------------------------------------------------------------- behaviour
def test_head_on_crowd_pair_does_not_crash(built):
    """§9h's K = 2, r = 4 m circle, where two straight drivers crash head-on: two crowd agents with the defaults, on the
    oracle with the host twin and the circle rule of evaluate(), both reach their goals."""
    from rl_collision_avoidance_b200.crowd import crowd_host
    sc, _, orc = make_pair('circle', num_worlds=1, gpu=False, seed=0, auto_reset=0, robots_per_world=2, radius=4.0)
    orc.reset_world()
    orc.reset_pose()
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=1, beams=512, auto_reset=0, seed=0)
    terminal = np.zeros(2, bool)
    first = [None, None]
    for _ in range(300):
        a = crowd_host(cfg, orc.pose, orc.goal, orc.meta, np.ones(2, np.uint8), np.zeros((2, 2), np.float32))
        a[terminal, 0] = 0.0
        orc.step(a)
        for i in range(2):
            if first[i] is None and orc.flags[i, 0]:
                first[i] = int(orc.flags[i, 2])
        terminal = orc.flags[:, 0] != 0
        if terminal.all():
            break
    assert first == [1, 1], first
