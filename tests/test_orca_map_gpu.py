"""The map-aware ORCA controllers on the H100 (DESIGN.md §9f): rlca_orca_action_map / rlca_nh_orca_action_map against
their host twins bit for bit on real tick states, on packed worlds next to walls of every robot count, and at the
candidate and line capacities; the all-free map against the map-blind entries; a wall between a robot and its goal in
the closed loop; evaluate() determinism and shard invariance; evaluate.py --orca-map end to end."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from helpers import random_actions
from rl_collision_avoidance_b200 import _lib
from test_orca_map import hand_world, map_cfg

pytestmark = pytest.mark.gpu


def _bits(t):
    return (t.cpu().numpy() if torch.is_tensor(t) else t).view(np.uint32)


def _params(nh):
    from rl_collision_avoidance_b200.orca import DEFAULTS, NH_DEFAULTS
    p = NH_DEFAULTS if nh else DEFAULTS
    return tuple(float(x) for x in p.values()), p


def _device_map(cfg, obs, pose, goal, meta, nh, args, tau_o, outputs=True):
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in (('pose', pose), ('goal', goal),
                                                                             ('meta', meta))}
    acc = torch.zeros_like(dev['pose'])
    st = _lib.EnvState(dev['pose'].data_ptr(), dev['goal'].data_ptr(), acc.data_ptr(), dev['meta'].data_ptr())
    n = len(pose)
    act = torch.full((n, 2), float('nan'), device='cuda')
    vel = torch.full((n, 2), float('nan'), device='cuda')
    status = torch.full((n,), -1, dtype=torch.int32, device='cuda')
    ptr = lambda t: C.c_void_p(t.data_ptr()) if outputs else None
    entry = _lib.load().rlca_nh_orca_action_map if nh else _lib.load().rlca_orca_action_map
    _lib.check(entry(C.byref(cfg), C.byref(st), obs.handle, *args, tau_o, C.c_void_p(act.data_ptr()), ptr(vel),
                     ptr(status), None))
    torch.cuda.synchronize()
    return act, vel, status


def _host_map(cfg, obs, pose, goal, meta, nh, p, tau_o):
    from rl_collision_avoidance_b200.orca import nh_orca_host, orca_host
    return (nh_orca_host if nh else orca_host)(cfg, pose, goal, meta, **p, obstacles=obs, obstacle_time_horizon=tau_o)


@pytest.mark.parametrize('nh', [False, True], ids=['orca-dd', 'nh-orca'])
@pytest.mark.parametrize('scenario, worlds, ticks', [('stage1', 171, 60), ('stage2', 8, 60), ('circle', 4, 40)])
def test_device_equals_host_on_tick_states(built, nh, scenario, worlds, ticks):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.orca import NhOrcaController, OrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=11, auto_reset=AUTO_RESET[scenario])
    env.reset_pose()
    rng = np.random.default_rng(worlds)
    for _ in range(ticks):
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda())
    ctrl = (NhOrcaController if nh else OrcaController)(env, obstacles=True)
    _, p = _params(nh)
    seen = set()
    for step in range(3):
        act = ctrl().clone()
        vel, st = ctrl.velocities().clone(), ctrl.status().clone()
        s = {k: v.cpu().numpy() for k, v in env.state.items()}
        h_act, h_vel, h_st = _host_map(env.cfg, ctrl.obstacles, s['pose'], s['goal'], s['meta'], nh, p,
                                       ctrl.obstacle_time_horizon)
        assert np.array_equal(_bits(act), _bits(h_act)), step
        assert np.array_equal(_bits(vel), _bits(h_vel)), step
        assert np.array_equal(st.cpu().numpy(), h_st), step
        seen |= set(np.unique(h_st).tolist())
        bare = torch.empty_like(act)
        entry = env.lib.rlca_nh_orca_action_map if nh else env.lib.rlca_orca_action_map
        _lib.check(entry(C.byref(env.cfg), C.byref(env._state_struct(env._cur)), ctrl.obstacles.handle, *ctrl.params,
                         ctrl.obstacle_time_horizon, C.c_void_p(bare.data_ptr()), None, None, env._stream()))
        torch.cuda.synchronize()
        assert np.array_equal(_bits(bare), _bits(h_act)), step
        env.control_vel(act)
    assert 0 in seen


def _wall_states(rng, R, W):
    from test_orca_map import _sample_states
    g, res, org = hand_world()
    return (g, res, org) + _sample_states(rng, g, res, org, R, W)


@pytest.mark.parametrize('nh', [False, True], ids=['orca-dd', 'nh-orca'])
def test_packed_worlds_next_to_walls(built, nh):
    """Every robot count from 1 to 64, robots packed next to the walls of the hand world (some inside them)."""
    from rl_collision_avoidance_b200.orca import ObstacleSet, obstacle_range
    args, p = _params(nh)
    seen = set()
    for R in range(1, 65):
        W = 3 if R % 8 else 2
        g, res, org, pose, goal, meta = _wall_states(np.random.default_rng(R), R, W)
        cfg = map_cfg(W, R, res, org)
        r_o = float(np.float32(p['radius']) + np.float32(p.get('tracking_error', 0.0)))
        obs = ObstacleSet(cfg, g, obstacle_range(cfg, r_o, 1.0))
        act, vel, st = _device_map(cfg, obs, pose, goal, meta, nh, args, 1.0)
        h_act, h_vel, h_st = _host_map(cfg, obs, pose, goal, meta, nh, p, 1.0)
        assert np.array_equal(_bits(act), _bits(h_act)), R
        assert np.array_equal(_bits(vel), _bits(h_vel)), R
        assert np.array_equal(st.cpu().numpy(), h_st), R
        seen |= set(h_st.tolist())
    assert 0 in seen and any(s & 1 for s in seen), seen


def _spread_world(rng, R, W):
    """Isolated cells 0.3 m apart at 0.1 m, tau_o = 1.3 s: bin lists of up to 478 candidates, robots among them."""
    g = np.zeros((90, 90), np.uint8)
    g[::3, ::3] = 254
    n = R * W
    pose = np.zeros((n, 4), np.float32)
    goal = np.zeros((n, 4), np.float32)
    meta = np.zeros((n, 4), np.int32)
    pose[:, 0:2], pose[:, 2] = rng.uniform(-3, 3, (n, 2)), rng.uniform(-np.pi, np.pi, n)
    goal[:, 0:2], goal[:, 2] = rng.uniform(-4, 4, (n, 2)), rng.uniform(0, 1, n)
    return g, 0.1, (45, 45), 1.3, pose, goal, meta


def _dense_world(rng, R, W):
    """tests/test_orca_map.dense_world: more obstacle lines than RLCA_ORCA_MAP_MAX_LINES near the centre."""
    from test_orca_map import DENSE_TAU_O, dense_states, dense_world
    g, res, org = dense_world()
    return (g, res, org, DENSE_TAU_O) + dense_states(rng, R, W)


@pytest.mark.parametrize('nh', [False, True], ids=['orca-dd', 'nh-orca'])
@pytest.mark.parametrize('world', ['candidates', 'lines'])
def test_candidate_and_line_capacities(built, nh, world):
    """'candidates': bin lists near RLCA_ORCA_MAP_MAX_CANDIDATES; 'lines': agents past RLCA_ORCA_MAP_MAX_LINES
    (status bit 2, the nearest 64 lines kept).  Device = host bit for bit, with and without the optional outputs."""
    from rl_collision_avoidance_b200.orca import ObstacleSet, obstacle_range
    args, p = _params(nh)
    R, W = 16, 5
    g, res, org, tau_o, pose, goal, meta = (_spread_world if world == 'candidates' else _dense_world)(
        np.random.default_rng(7), R, W)
    cfg = map_cfg(W, R, res, org)
    r_o = float(np.float32(p['radius']) + np.float32(p.get('tracking_error', 0.0)))
    obs = ObstacleSet(cfg, g, obstacle_range(cfg, r_o, tau_o))
    _, _, longest = obs.segments()
    assert longest > 384, longest
    for outputs in (True, False):
        act, vel, st = _device_map(cfg, obs, pose, goal, meta, nh, args, tau_o, outputs)
        h_act, h_vel, h_st = _host_map(cfg, obs, pose, goal, meta, nh, p, tau_o)
        assert np.array_equal(_bits(act), _bits(h_act))
        if outputs:
            assert np.array_equal(_bits(vel), _bits(h_vel))
            assert np.array_equal(st.cpu().numpy(), h_st)
    if world == 'lines':
        assert np.mean((h_st & 4) != 0) >= 0.25, np.unique(h_st, return_counts=True)
    else:
        assert np.any(h_st == 0) and np.any(h_st & 2), np.unique(h_st)


@pytest.mark.parametrize('nh', [False, True], ids=['orca-dd', 'nh-orca'])
def test_all_free_map_equals_map_blind_on_device(built, nh):
    from helpers import orca_sweep_states
    from rl_collision_avoidance_b200.orca import ObstacleSet
    args, p = _params(nh)
    for (seed, R, W, side), (pose, goal, meta) in orca_sweep_states(range(1, 3), p['neighbour_dist']):
        cfg = map_cfg(W, R, 0.2, (20, 15))
        obs = ObstacleSet(cfg, np.zeros((30, 40), np.uint8), 2.0)
        act, vel, st = _device_map(cfg, obs, pose, goal, meta, nh, args, 1.0)
        dev = {k: torch.from_numpy(v).cuda() for k, v in (('pose', pose), ('goal', goal), ('meta', meta))}
        acc = torch.zeros_like(dev['pose'])
        es = _lib.EnvState(dev['pose'].data_ptr(), dev['goal'].data_ptr(), acc.data_ptr(), dev['meta'].data_ptr())
        b_act, b_vel, b_st = torch.empty_like(act), torch.empty_like(vel), torch.empty_like(st)
        entry = _lib.load().rlca_nh_orca_action if nh else _lib.load().rlca_orca_action
        _lib.check(entry(C.byref(cfg), C.byref(es), *args, C.c_void_p(b_act.data_ptr()),
                         C.c_void_p(b_vel.data_ptr()), C.c_void_p(b_st.data_ptr()), None))
        torch.cuda.synchronize()
        assert np.array_equal(_bits(act), _bits(b_act)) and np.array_equal(_bits(vel), _bits(b_vel))
        assert np.array_equal(st.cpu().numpy(), b_st.cpu().numpy())


def _wall_scenario():
    """Two robots swapping across a 6 m circle with a 1.2 m wall across the middle, off-centre."""
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.worldfile import WorldMap
    g = np.zeros((100, 100), np.uint8)
    g[46:58, 48:52] = 254                               # x in [-0.2, 0.2], y in [-0.4, 0.8]
    m = WorldMap(cells=g, resolution=0.1, origin_cx=50, origin_cy=50, init_poses=np.zeros((0, 3)), name='wall')
    return make_scenario('circle', map_=m, robots_per_world=2, radius=3.0)


@pytest.mark.parametrize('nh', [False, True], ids=['orca-dd', 'nh-orca'])
def test_wall_between_robot_and_goal_closed_loop(built, nh):
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController, OrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    Ctrl = NhOrcaController if nh else OrcaController
    out = {}
    for aware in (False, True):
        env = StageWorld(512, scenario=_wall_scenario(), num_worlds=2, seed=0, auto_reset=0)
        out[aware] = evaluate(env, Ctrl(env, obstacles=aware), 1, max_ticks=400, check_every=10)['metrics']
    assert out[False]['crashed'] > 0, out[False]
    assert out[True]['crashed'] == 0, out[True]


def test_evaluate_with_map_is_deterministic_and_shard_invariant(built):
    from rl_collision_avoidance_b200.evaluation import evaluate, totals
    from rl_collision_avoidance_b200.orca import NhOrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=8, seed=5, auto_reset=1)
    ctrl = NhOrcaController(env, obstacles=True)
    a = evaluate(env, ctrl, 2, max_ticks=320)
    b = evaluate(env, ctrl, 2, max_ticks=320)
    assert np.array_equal(a['totals'].view(np.uint64), b['totals'].view(np.uint64))
    del env, ctrl
    parts = []
    for off in (0, 4):
        e = StageWorld(512, scenario='stage1', num_worlds=4, seed=5, auto_reset=1, world_offset=off)
        parts.append(evaluate(e, NhOrcaController(e, obstacles=True), 2, max_ticks=320)['partials'])
    sharded = np.concatenate(parts)
    assert np.array_equal(sharded.view(np.uint64), a['partials'].view(np.uint64))
    assert np.array_equal(totals(sharded).view(np.uint64), a['totals'].view(np.uint64))
    assert a['totals'][0] > 0


def test_evaluate_py_nh_orca_map(built, tmp_path, capsys):
    import evaluate as drv
    out = tmp_path / 'nhmap.json'
    drv.main(['--scenario', 'stage1', '--baseline', 'nh-orca', '--orca-map', '--num-worlds', '2', '--max-ticks', '200',
              '--json', str(out)])
    d = json.loads(out.read_text())
    assert d['controller'] == 'nh-orca+map' and d['robots'] == 48
    assert capsys.readouterr().out.startswith('nh-orca+map  stage1')
