"""The NH-ORCA controller on the H100 (DESIGN.md §9e): rlca_nh_orca_action against rlca_nh_orca_action_host bit for bit
on states from real ticks and on hand-built packed worlds of every robot count, the closed loop on the K = 2 circle
swap, and evaluate() / evaluate.py with the controller."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from helpers import orca_cfg, random_actions
from rl_collision_avoidance_b200 import _lib

pytestmark = pytest.mark.gpu


def _run_ticks(env, ticks, seed):
    rng = np.random.default_rng(seed)
    for _ in range(ticks):
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda())


def _bits(t):
    return (t.cpu().numpy() if torch.is_tensor(t) else t).view(np.uint32)


@pytest.mark.parametrize('scenario, worlds, K, ticks', [('stage1', 171, None, 60), ('stage2', 8, None, 60),
                                                        ('circle', 4, None, 40), ('circle', 3, 64, 40)])
def test_device_equals_host_bit_for_bit(built, scenario, worlds, K, ticks):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.orca import NhOrcaController, nh_orca_host
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('circle', robots_per_world=K, radius=8.0) if K else make_scenario(scenario)
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=11, auto_reset=AUTO_RESET[scenario])
    env.reset_pose()
    _run_ticks(env, ticks, seed=worlds)
    ctrl = NhOrcaController(env)
    statuses = set()
    for step in range(3):                      # three states: after the random ticks, then under NH-ORCA
        act = ctrl().clone()
        vel, st = ctrl.velocities().clone(), ctrl.status().clone()
        s = {k: v.cpu().numpy() for k, v in env.state.items()}
        h_act, h_vel, h_st = nh_orca_host(env.cfg, s['pose'], s['goal'], s['meta'], *ctrl.params)
        assert np.array_equal(_bits(act), _bits(h_act)), step
        assert np.array_equal(_bits(vel), _bits(h_vel)), step
        assert np.array_equal(st.cpu().numpy(), h_st), step
        statuses |= set(np.unique(h_st).tolist())
        # without the optional outputs: the same actions
        bare = torch.empty_like(act)
        _lib.check(env.lib.rlca_nh_orca_action(C.byref(env.cfg), C.byref(env._state_struct(env._cur)), *ctrl.params,
                                               C.c_void_p(bare.data_ptr()), None, None, env._stream()))
        assert np.array_equal(_bits(bare), _bits(h_act)), step
        env.control_vel(act)
    assert 0 in statuses


def _packed(rng, R, W, side, inner):
    """W worlds of R robots: robots 0-31 of each world in a side x side box, robots 32 on in an inner x inner box at
    its centre (as tests/test_orca_dense_gpu.py builds them for ORCA-DD)."""
    n = R * W
    r = np.arange(n) % R
    half = np.where(r < 32, side, inner)[:, None] / 2
    xy = rng.uniform(-1, 1, (n, 2)) * half
    pose = np.zeros((n, 4), np.float32)
    goal = np.zeros((n, 4), np.float32)
    meta = np.zeros((n, 4), np.int32)
    pose[:, 0:2], pose[:, 2] = xy, rng.uniform(-np.pi, np.pi, n)
    goal[:, 0:2], goal[:, 2] = xy + rng.uniform(-10, 10, (n, 2)), rng.uniform(0, 1, n)
    meta[:, 2] = rng.random(n) < 0.1
    return pose, goal, meta


# R * W is not a multiple of the 8 agents of a CTA except at R = 32 and 64
ROBOT_COUNTS = [(1, 5, 1.0, 1.0), (2, 3, 1.0, 1.0), (3, 5, 1.5, 1.5), (31, 3, 4.0, 4.0), (32, 1, 4.0, 4.0),
                (33, 3, 4.0, 4.0), (34, 3, 6.0, 2.0), (63, 2, 6.0, 3.0), (64, 2, 6.0, 3.0)]


def test_packed_worlds_device_equals_host(built):
    from rl_collision_avoidance_b200.orca import NH_DEFAULTS, nh_orca_host
    seen = set()
    for R in range(1, 65):
        W, side, inner = next(((w, s, i) for r, w, s, i in ROBOT_COUNTS if r >= R), (2, 6.0, 3.0))
        pose, goal, meta = _packed(np.random.default_rng(R), R, W, side, inner)
        cfg = orca_cfg(W, R)
        p = dict(NH_DEFAULTS, neighbour_dist=2 * side)
        dev = {k: torch.from_numpy(v).cuda() for k, v in (('pose', pose), ('goal', goal), ('meta', meta))}
        acc = torch.zeros_like(dev['pose'])
        st = _lib.EnvState(dev['pose'].data_ptr(), dev['goal'].data_ptr(), acc.data_ptr(), dev['meta'].data_ptr())
        n = R * W
        act = torch.full((n, 2), float('nan'), device='cuda')
        vel = torch.full((n, 2), float('nan'), device='cuda')
        status = torch.full((n,), -1, dtype=torch.int32, device='cuda')
        ptr = lambda t: C.c_void_p(t.data_ptr())
        args = (p['radius'], p['neighbour_dist'], p['time_horizon'], p['tracking_error'], p['heading_time'])
        _lib.check(_lib.load().rlca_nh_orca_action(C.byref(cfg), C.byref(st), *args, ptr(act), ptr(vel),
                                                   ptr(status), None))
        torch.cuda.synchronize()
        h_act, h_vel, h_st = nh_orca_host(cfg, pose, goal, meta, **p)
        assert np.array_equal(_bits(act), _bits(h_act)), R
        assert np.array_equal(_bits(vel), _bits(h_vel)), R
        assert np.array_equal(status.cpu().numpy(), h_st), R
        seen |= set(h_st.tolist())
    assert seen == {0, 1}


@pytest.mark.parametrize('K', [2])
def test_circle_swap_closed_loop(built, K):
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=make_scenario('circle', robots_per_world=K, radius=4.0), num_worlds=2, seed=0,
                     auto_reset=0)
    out = evaluate(env, NhOrcaController(env), 1, max_ticks=600, check_every=10)
    m = out['metrics']
    assert m['reached'] == env.N and m['crashed'] == 0 and m['timed_out'] == 0 and m['unfinished'] == 0, m


def test_evaluate_with_nh_orca_is_deterministic_and_shard_invariant(built):
    from rl_collision_avoidance_b200.evaluation import evaluate, totals
    from rl_collision_avoidance_b200.orca import NhOrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=8, seed=5, auto_reset=1)
    ctrl = NhOrcaController(env)
    a = evaluate(env, ctrl, 2, max_ticks=320)
    b = evaluate(env, ctrl, 2, max_ticks=320)
    assert np.array_equal(a['totals'].view(np.uint64), b['totals'].view(np.uint64))
    del env, ctrl
    parts = []
    for off in (0, 4):
        e = StageWorld(512, scenario='stage1', num_worlds=4, seed=5, auto_reset=1, world_offset=off)
        parts.append(evaluate(e, NhOrcaController(e), 2, max_ticks=320)['partials'])
    sharded = np.concatenate(parts)
    assert np.array_equal(sharded.view(np.uint64), a['partials'].view(np.uint64))
    assert np.array_equal(totals(sharded).view(np.uint64), a['totals'].view(np.uint64))
    assert a['totals'][0] > 0


def test_evaluate_py_baseline_nh_orca(built, tmp_path, capsys):
    import evaluate as drv
    out = tmp_path / 'nh.json'
    drv.main(['--scenario', 'circle', '--baseline', 'nh-orca', '--num-worlds', '2', '--circle-robots', '6',
              '--circle-radius', '4', '--max-ticks', '400', '--json', str(out)])
    d = json.loads(out.read_text())
    assert d['controller'] == 'nh-orca' and d['robots'] == 12
    assert d['metrics']['episodes'] + d['metrics']['unfinished'] == 12
    assert capsys.readouterr().out.startswith('nh-orca  circle')
