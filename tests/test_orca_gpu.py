"""The ORCA-DD controller on the H100: rlca_orca_action against rlca_orca_action_host bit for bit on states from real
ticks, the closed loop on small circle swaps, and evaluate() / evaluate.py with the controller."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from helpers import random_actions
from rl_collision_avoidance_b200 import _lib

pytestmark = pytest.mark.gpu


def _run_ticks(env, ticks, seed):
    rng = np.random.default_rng(seed)
    for _ in range(ticks):
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda())


@pytest.mark.parametrize('scenario, worlds, K, ticks', [('stage1', 171, None, 60), ('stage2', 8, None, 60),
                                                        ('circle', 4, None, 40), ('circle', 3, 64, 40)])
def test_device_equals_host_bit_for_bit(built, scenario, worlds, K, ticks):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.orca import OrcaController, orca_host
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('circle', robots_per_world=K, radius=8.0) if K else make_scenario(scenario)
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=11, auto_reset=AUTO_RESET[scenario])
    env.reset_pose()
    _run_ticks(env, ticks, seed=worlds)
    ctrl = OrcaController(env)
    statuses = set()
    for step in range(3):                      # three states: after the random ticks, then under ORCA-DD
        act = ctrl().clone()
        vel, st = ctrl.velocities().clone(), ctrl.status().clone()
        s = {k: v.cpu().numpy() for k, v in env.state.items()}
        h_act, h_vel, h_st = orca_host(env.cfg, s['pose'], s['goal'], s['meta'], *ctrl.params)
        assert np.array_equal(act.cpu().numpy().view(np.uint32), h_act.view(np.uint32)), step
        assert np.array_equal(vel.cpu().numpy().view(np.uint32), h_vel.view(np.uint32)), step
        assert np.array_equal(st.cpu().numpy(), h_st), step
        statuses |= set(np.unique(h_st).tolist())
        # without the optional outputs: the same actions
        bare = torch.empty_like(act)
        _lib.check(env.lib.rlca_orca_action(C.byref(env.cfg), C.byref(env._state_struct(env._cur)), *ctrl.params,
                                            C.c_void_p(bare.data_ptr()), None, None, env._stream()))
        assert np.array_equal(bare.cpu().numpy().view(np.uint32), h_act.view(np.uint32)), step
        env.control_vel(act)
    assert 0 in statuses


@pytest.mark.parametrize('K', [2])
def test_circle_swap_closed_loop(built, K):
    # K = 4 at 4 m does not complete: the four robots stall round the centre (DESIGN.md §9d)
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import OrcaController
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=make_scenario('circle', robots_per_world=K, radius=4.0), num_worlds=2, seed=0,
                     auto_reset=0)
    out = evaluate(env, OrcaController(env), 1, max_ticks=600, check_every=10)
    m = out['metrics']
    assert m['reached'] == env.N and m['crashed'] == 0 and m['timed_out'] == 0 and m['unfinished'] == 0, m


def test_evaluate_with_orca_is_deterministic_and_shard_invariant(built):
    from rl_collision_avoidance_b200.evaluation import evaluate, totals
    from rl_collision_avoidance_b200.orca import OrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=8, seed=5, auto_reset=1)
    ctrl = OrcaController(env)
    a = evaluate(env, ctrl, 2, max_ticks=320)
    b = evaluate(env, ctrl, 2, max_ticks=320)
    assert np.array_equal(a['totals'].view(np.uint64), b['totals'].view(np.uint64))
    del env, ctrl
    parts = []
    for off in (0, 4):
        e = StageWorld(512, scenario='stage1', num_worlds=4, seed=5, auto_reset=1, world_offset=off)
        parts.append(evaluate(e, OrcaController(e), 2, max_ticks=320)['partials'])
    sharded = np.concatenate(parts)
    assert np.array_equal(sharded.view(np.uint64), a['partials'].view(np.uint64))
    assert np.array_equal(totals(sharded).view(np.uint64), a['totals'].view(np.uint64))
    assert a['totals'][0] > 0


def test_evaluate_py_baseline_orca(built, tmp_path):
    import evaluate as drv
    out = tmp_path / 'orca.json'
    drv.main(['--scenario', 'circle', '--baseline', 'orca', '--num-worlds', '2', '--circle-robots', '6',
              '--circle-radius', '4', '--max-ticks', '400', '--json', str(out)])
    d = json.loads(out.read_text())
    assert d['controller'] == 'orca-dd' and d['robots'] == 12
    assert d['metrics']['episodes'] + d['metrics']['unfinished'] == 12
