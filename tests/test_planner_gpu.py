"""The global planner on the device (DESIGN.md §9w): rlca_plan_fields, rlca_plan_waypoints and rlca_plan_track against
their host twins bit for bit at the evaluation shapes and after every tick of a stage-1 rollout, and evaluate() /
evaluate.py with the planner, deterministic and shard-invariant."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import random_actions

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGE2 = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _scenario(name):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    if name == 'arena':
        return make_scenario('arena', robots_per_world=16, arenas=64)
    return make_scenario(name)


def _env(sc, W, seed=0, world_offset=0, auto_reset=0):
    from rl_collision_avoidance_b200.stage_world import StageWorld
    return StageWorld(512, scenario=sc, num_worlds=W, seed=seed, auto_reset=auto_reset, world_offset=world_offset)


def _compare(env, planner, hs, steer=True):
    """The device planner state against the host twins run on the same env state (hs carried along)."""
    from rl_collision_avoidance_b200.planner import fields_host, waypoints_host
    torch.cuda.synchronize()
    st = env.state
    pose, goal = st['pose'].cpu().numpy(), st['goal'].cpu().numpy()
    gs = env.gs.cpu().numpy()
    fields_host(env.cfg, planner.tables, hs, goal)
    entry = planner.entry.cpu().numpy()
    assert _same(entry, hs.entry)
    lst = planner.list.cpu().numpy()
    assert sorted(lst[1:1 + lst[0]]) == list(hs.replanned())
    rect = planner.rect.cpu().numpy()
    field = planner.field.cpu().numpy().view(np.uint32)
    for a in np.nonzero(entry >= 0)[0]:
        assert _same(rect[a], hs.rect[a])
        x0, y0, x1, y1 = rect[a]
        A = (x1 - x0 + 1) * (y1 - y0 + 1)
        assert _same(field[a, :A], hs.field[a, :A]), a
    if steer:
        out = waypoints_host(env.cfg, planner.tables, hs, pose, goal, gs)
        status = planner.status().cpu().numpy()
        assert _same(status, hs.status)
        assert _same(planner.gs.cpu().numpy(), out)
        assert _same(planner.gs.cpu().numpy()[status != 1], gs[status != 1])
        assert _same(planner.status_count.cpu().numpy(), hs.status_count)
        return status
    return None


@pytest.mark.parametrize('name, W', [('stage1', 171), ('stage2', 24), ('arena', 1024)])
def test_kernels_equal_host_twins(built, name, W):
    from rl_collision_avoidance_b200.planner import HostState, Planner
    sc = _scenario(name)
    env = _env(sc, W, seed=3, auto_reset={'stage1': 1, 'stage2': 2, 'arena': 0}[name])
    env.reset_world()
    env.reset_pose()
    if sc.layout is not None:
        env.random_layout()
    planner = Planner(env)
    hs = HostState(env.cfg, planner.tables)
    planner.update()
    status = _compare(env, planner, hs)
    assert (status == 0).any()
    planner.update()                                    # nothing changed: nothing re-planned
    torch.cuda.synchronize()
    assert int(planner.list[0]) == 0
    _compare(env, planner, hs)


def test_rollout_stage1_every_tick(built):
    """200 ticks of stage 1 with re-spawns: fields, waypoints and the geodesic tracker equal their twins after every
    tick."""
    from rl_collision_avoidance_b200.evaluation import EpisodeTracker
    from rl_collision_avoidance_b200.planner import HostState, Planner, track_host
    sc = _scenario('stage1')
    env = _env(sc, 8, seed=4, auto_reset=1)
    env.reset_world()
    env.reset_pose()
    tracker = EpisodeTracker(env, 4)
    tracker.reset()
    planner = Planner(env)
    planner.attach(tracker)
    hs = HostState(env.cfg, planner.tables, episodes=4)
    planner.update()
    _compare(env, planner, hs)
    track_host(env.cfg, planner.tables, hs, env.state['acc'].cpu().numpy())
    rng = np.random.default_rng(0)
    replans = 0
    for t in range(200):
        meta_in = env.state['meta'].cpu().numpy()
        closed, count = tracker.closed.cpu().numpy(), tracker.count.cpu().numpy()
        a = random_actions(rng, env.N)
        a[:, 0] = np.abs(a[:, 0])
        env.control_vel(torch.from_numpy(a).cuda())
        planner.update(env.flags)
        _compare(env, planner, hs)
        track_host(env.cfg, planner.tables, hs, env.state['acc'].cpu().numpy(), meta_in, env.flags.cpu().numpy(),
                   closed, count)
        assert _same(planner.length.cpu().numpy(), hs.length) and _same(planner.records.cpu().numpy(), hs.records)
        tracker.track()
        replans += int(planner.list[0])
    assert replans > 0 and int(tracker.count.sum()) > 0


def test_stage2_group_respawn_replans_only_random_goals(built):
    """Stage 2's group re-spawn puts a table robot back on its table goal: only the random-goal rows re-plan."""
    from rl_collision_avoidance_b200.planner import Planner
    sc = _scenario('stage2')
    env = _env(sc, 2, seed=1, auto_reset=2)
    env.reset_world()
    env.reset_pose()
    planner = Planner(env, steer=False)
    planner.update()
    rng = np.random.default_rng(1)
    table = np.tile(sc.goal_tab[:, 2] == 0, 2)
    seen = 0
    for t in range(300):
        a = random_actions(rng, env.N)
        env.control_vel(torch.from_numpy(a).cuda())
        planner.update(env.flags)
        torch.cuda.synchronize()
        lst = planner.list.cpu().numpy()
        rows = lst[1:1 + lst[0]]
        respawned = env.flags[:, 3].cpu().numpy() != 0
        assert not table[rows].any()
        seen += int(respawned[table].sum())
    assert seen > 0


def _controllers(env, kind):
    from rl_collision_avoidance_b200.crowd import Crowd
    from rl_collision_avoidance_b200.dwa import DwaController
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    kw = {}
    if kind == 'dwa':
        return DwaController(env), kw
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(STAGE2, map_location='cuda'))
    if kind == 'crowd':
        kw['crowd'] = Crowd(env, non_cooperative_mask(env.num_env, env.num_worlds, 2), obstacles=True)
    return pol, kw


@pytest.mark.parametrize('name, kind', [('arena', 'policy'), ('stage2', 'policy'), ('arena', 'dwa'),
                                        ('arena', 'crowd')])
def test_evaluate_with_planner_is_deterministic_and_shard_invariant(built, name, kind):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate
    from rl_collision_avoidance_b200.planner import Planner
    from rl_collision_avoidance_b200.scenarios import make_scenario, random_max_ticks
    sc = make_scenario('arena', robots_per_world=8, arenas=16) if name == 'arena' else make_scenario('stage2')
    ticks = random_max_ticks(sc.layout.side) if name == 'arena' else 2 * (sc.timeout + 1)
    W = 8 if name == 'arena' else 4

    def run(W, wo):
        env = _env(sc, W, seed=5, world_offset=wo, auto_reset=AUTO_RESET[name])
        pol, kw = _controllers(env, kind)
        return evaluate(env, pol, 2 if name == 'stage2' else 1, ticks, check_every=50, progress={},
                        planner=Planner(env), **kw)

    a, b = run(W, 0), run(W, 0)
    for k in ('partials', 'geodesic_partials', 'progress_partials'):
        assert np.array_equal(a[k], b[k]), k
    assert a['planner'] == b['planner'] and a['planner']['waypoint'] > 0
    assert a['geodesic']['reached'] > 0 or a['metrics']['reached'] == 0
    parts = [run(W // 2, 0), run(W - W // 2, W // 2)]
    for k in ('partials', 'geodesic_partials'):
        assert np.array_equal(np.concatenate([p[k] for p in parts]), a[k]), k
    if kind == 'crowd':
        assert set(a['geodesic_by_role']) == {'cooperative', 'crowd'}


def test_geodesic_with_nh_orca_map(built):
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController
    from rl_collision_avoidance_b200.planner import Planner
    from rl_collision_avoidance_b200.scenarios import make_scenario, random_max_ticks
    sc = make_scenario('arena', robots_per_world=8, arenas=16)
    env = _env(sc, 8, seed=2)
    out = evaluate(env, NhOrcaController(env, obstacles=True), 1, random_max_ticks(sc.layout.side),
                   planner=Planner(env, steer=False))
    assert 'planner' not in out and out['geodesic']['reached'] > 0
    assert out['geodesic']['reached'] <= out['metrics']['reached']
    assert out['geodesic']['mean_length'] > 0


def test_evaluate_cli_planner_json_is_reproducible(built, tmp_path):
    import evaluate
    outs = []
    for i in range(2):
        path = tmp_path / f'{i}.json'
        evaluate.main(['--scenario', 'arena', '--policy', STAGE2, '--num-worlds', '16', '--arena-robots', '8',
                       '--arena-count', '16', '--seed', '2', '--planner', '--timeouts', '--json', str(path)])
        outs.append(json.loads(path.read_text()))
    for k in ('metrics', 'partials', 'planner', 'geodesic'):
        assert outs[0][k] == outs[1][k], k
    res = outs[0]
    assert res['planner']['steer'] is True and res['geodesic']['metrics']['reached'] >= 0
    assert res['args']['planner'] is True
