"""Progress metrics on the device (csrc/rlca_progress.cu, DESIGN.md §9o): rlca_progress_track against its host twin
bit for bit on every scenario and episode mechanic, scripted controllers with their expected causes, consistency with
the episode tracker, evaluate() with the option on against the recorded partials, determinism and shard invariance,
the split by role, and evaluate.py --timeouts end to end."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from helpers import random_actions
from rl_collision_avoidance_b200.scenarios import make_scenario

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cpu'))
    return pol


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _np(t):
    return t.cpu().numpy()


def _host_state(N, E):
    return dict(running=np.zeros((N, 4), np.float32), counters=np.zeros((N, 4), np.int32),
                records=np.zeros((N, E, 4), np.float32), causes=np.zeros((N, E), np.uint8))


def _check_against_tracker(tr, pt, E):
    """Causes exactly on the time-outs; per world the causes add up to the tracker's time-outs and unfinished."""
    cnt = np.minimum(_np(tr.count), E)
    res, causes = _np(tr.records), _np(pt.causes)
    for a in range(len(cnt)):
        assert np.array_equal(causes[a, :cnt[a]] != 0, res[a, :cnt[a], 0] == 3), a
        assert not causes[a, cnt[a]:].any() and not _np(pt.records)[a, cnt[a]:].any()
    ev, pp = tr.partials(), pt.partials()
    assert np.array_equal(pp[:, 0:3].sum(1), ev[:, 2]) and np.array_equal(pp[:, 7:10].sum(1), ev[:, 3])
    assert np.array_equal(pp[:, 16], ev[:, 0])
    return ev, pp


# (id, scenario keywords, auto_reset, worlds)
TRACK_CASES = [
    ('stage1', dict(name='stage1'), 1, 2),
    ('stage2', dict(name='stage2'), 2, 2),
    ('circle16', dict(name='circle', robots_per_world=16, radius=4.0), 0, 2),
    ('random2', dict(name='random', robots_per_world=2, side=3.0, separation=0.8, min_travel=1.5, timeout=60), 0, 6),
    ('random8', dict(name='random', robots_per_world=8, side=5.0, separation=0.8, min_travel=2.0, timeout=80), 0, 3),
    ('random64', dict(name='random', robots_per_world=64, side=14.0, separation=0.8, min_travel=5.0, timeout=100), 0,
     1),
]


@pytest.mark.parametrize('case', TRACK_CASES, ids=[c[0] for c in TRACK_CASES])
def test_device_track_equals_host_twin(built, case):
    """300 random-action ticks (every third robot standing still): running state, records and causes of the kernel
    equal rlca_progress_track_host fed with the same poses, flags and tracker state; the reduction equals the host's."""
    from rl_collision_avoidance_b200.evaluation import EpisodeTracker, ProgressTracker, progress_reduce_host, \
        progress_track_host
    from rl_collision_avoidance_b200.stage_world import StageWorld
    _, kw, auto_reset, worlds = case
    kw = dict(kw)
    sc = make_scenario(kw.pop('name'), **kw)
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=31, auto_reset=auto_reset)
    env.reset_pose()
    if sc.layout is not None:
        env.random_layout()
    E = 3
    params = {'window': 15, 'still_dist': 0.01, 'block_dist': 1.0}
    tr = EpisodeTracker(env, E)
    pt = ProgressTracker(env, tr, params)
    host = _host_state(env.N, E)
    rng = np.random.default_rng(32)
    seen_respawn = seen_near = 0
    for t in range(300):
        a = random_actions(rng, env.N)
        a[::3, 0] = 0.0
        pose_in, meta_in = _np(env.state['pose']), _np(env.state['meta'])
        env.control_vel(torch.from_numpy(a).cuda())
        closed, count = _np(tr.closed), _np(tr.count)
        pt.track()
        tr.track()
        flags = _np(env.flags)
        progress_track_host(env.cfg, params, pose_in, meta_in, _np(env.state['pose']), flags, closed, count, host)
        seen_respawn += int(flags[:, 3].sum())
        seen_near += int((host['running'][:, 3] != 0).sum())
        if t % 50 == 49 or t < 3:
            for k in host:
                assert _bits_equal(_np(getattr(pt, k)), host[k]), (t, k)
    assert (seen_respawn > 0) == (auto_reset == 1) or auto_reset == 2
    ev, pp = _check_against_tracker(tr, pt, E)
    assert ev[:, 2].sum() > 0 or ev[:, 3].sum() > 0
    want = progress_reduce_host(env.cfg, params, host, _np(tr.records), _np(tr.count), _np(tr.open))
    assert _bits_equal(pp, want)
    if sc.robots_per_world >= 8:
        assert seen_near > 0, 'no robot near in the run'


def _scripted(K, worlds, timeout, window, action, place=None, separation=3.0, min_travel=4.0, side=10.0,
              all_time_out=True):
    """Random layouts with starts `separation` apart and a `timeout`-tick budget, every robot driven by action(env)
    for timeout + 5 ticks; returns (episode partials, progress partials, causes of the recorded episodes)."""
    from rl_collision_avoidance_b200.evaluation import EpisodeTracker, ProgressTracker
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('random', robots_per_world=K, side=side, separation=separation, min_travel=min_travel,
                       timeout=timeout)
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=41, auto_reset=0)
    env.reset_pose()
    env.random_layout()
    if place is not None:
        place(env)
    tr = EpisodeTracker(env, 1)
    pt = ProgressTracker(env, tr, {'window': window})
    for _ in range(timeout + 5):
        env.control_vel(action(env))
        pt.track()
        tr.track()
    ev, pp = _check_against_tracker(tr, pt, 1)
    assert ev[:, 2].sum() == env.N or not all_time_out, 'every robot should time out'
    return ev, pp, _np(pt.causes)[:, 0]


def test_scripted_controllers_give_the_expected_causes(built):
    from rl_collision_avoidance_b200.orca import NonCooperative
    const = lambda v, w: (lambda env: torch.tensor([[v, w]], device='cuda').repeat(env.N, 1))
    # v = 0: frozen, nobody within 1 m
    _, _, causes = _scripted(4, 16, 80, 50, const(0.0, 0.0))
    assert (causes == 1).all(), np.unique(causes)
    # v = 1, w = 1: a 1 m circle, moving and never closer: stalled
    _, _, causes = _scripted(2, 32, 200, 50, const(1.0, 1.0), separation=5.0)
    assert (causes == 2).all(), np.unique(causes)
    # straight to the goal, a budget shorter than the trip: slow (two straight paths may cross: a crash is no time-out)
    drivers = {}

    def straight(env):
        if 'nc' not in drivers:
            drivers['nc'] = NonCooperative(env, np.ones(env.N, np.uint8))
        return drivers['nc'].apply(torch.zeros(env.N, 2, device='cuda'))

    _, pp, causes = _scripted(2, 32, 55, 40, straight, separation=4.0, min_travel=6.5, all_time_out=False)
    slow = (causes & 3) == 3                    # two paths may cross: a crash (cause 0) or a robot near (+ 4)
    assert slow[causes != 0].all() and slow.sum() >= len(causes) // 2, np.unique(causes)
    assert pp[:, 5].sum() / pp[:, 4].sum() > 1.5                    # the goals are still far

    # two robots 0.7 m apart, v = 0: frozen + robot near
    def pair(env):
        pose = env.state['pose'][:, 0:3].clone()
        pose[1::2] = pose[0::2] + torch.tensor([0.7, 0.0, 0.0], device='cuda')
        env.control_pose(pose)

    _, _, causes = _scripted(2, 16, 60, 50, const(0.0, 0.0), place=pair, separation=3.0, min_travel=3.0)
    assert (causes == 5).all(), np.unique(causes)


def _golden_run(name, **kw):
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController, OrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    scenario, worlds, seed, who, episodes, max_ticks, check_every = make_golden_eval.RUNS[name]
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])
    policy = OrcaController(env) if who == 'orca' else NhOrcaController(env, obstacles=True) if who == 'nh-orca' \
        else _policy(who, env.N)
    return env, evaluate(env, policy, episodes, max_ticks, check_every=check_every, **kw)


def test_evaluate_with_progress_keeps_the_recorded_partials(built):
    """Every run of tests/golden/eval_partials.npz with the option on, next to --safety: the same partials and ticks
    bit for bit, the same safety partials as with --safety alone, the device reduction equal to the host's."""
    from rl_collision_avoidance_b200.evaluation import PROGRESS_COLUMNS, progress_reduce_host
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_partials.npz'))
    for name in make_golden_eval.RUNS:
        env, out = _golden_run(name, safety=0.1, progress={})
        assert out['ticks'] == int(g['ticks_' + name]), name
        assert np.array_equal(out['partials'].view(np.uint64), g['partials_' + name].view(np.uint64)), name
        _, alone = _golden_run(name, safety=0.1)
        assert _bits_equal(out['safety_partials'], alone['safety_partials']), name
        assert not any(k.startswith('progress') for k in alone)
        pp, tr, pt = out['progress_partials'], out['tracker'], out['progress_tracker']
        assert pp.shape == (env.num_worlds, len(PROGRESS_COLUMNS))
        st = {k: _np(getattr(pt, k)) for k in ('running', 'counters', 'records', 'causes')}
        host = progress_reduce_host(env.cfg, pt.params, st, _np(tr.records), _np(tr.count), _np(tr.open))
        assert _bits_equal(pp, host), name
        assert np.array_equal(pp[:, 0:3].sum(1), out['partials'][:, 2]), name
        assert np.array_equal(pp[:, 7:10].sum(1), out['partials'][:, 3]), name
        assert np.array_equal(pp[:, 16], out['partials'][:, 0]), name


def test_progress_is_deterministic_shard_invariant_and_split_by_role(built):
    from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask, progress_totals
    from rl_collision_avoidance_b200.orca import NhOrcaController, NonCooperative
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('random', robots_per_world=8, side=6.0, separation=0.8, min_travel=3.0)

    def run(W, off, progress=None):
        env = StageWorld(512, scenario=sc, num_worlds=W, seed=5, auto_reset=0, world_offset=off)
        return evaluate(env, NhOrcaController(env, obstacles=True), 1, 60, progress=progress)

    p = {'window': 10}
    a, b = run(8, 0, p), run(8, 0, p)
    assert _bits_equal(a['progress_partials'], b['progress_partials']) and _bits_equal(a['partials'], b['partials'])
    parts = np.concatenate([run(4, off, p)['progress_partials'] for off in (0, 4)])
    assert _bits_equal(parts, a['progress_partials'])
    assert _bits_equal(progress_totals(parts), a['progress_totals'])
    assert a['progress']['unfinished'] > 0
    plain = run(8, 0)
    assert _bits_equal(plain['partials'], a['partials']) and plain['ticks'] == a['ticks']
    # roles: stage2.pth among non-cooperative robots on the circle
    sc = make_scenario('circle', robots_per_world=12, radius=4.0)
    env = StageWorld(512, scenario=sc, num_worlds=6, seed=2, auto_reset=0)
    nc = NonCooperative(env, non_cooperative_mask(12, 6, 2))
    out = evaluate(env, _policy('stage2.pth', env.N), 1, 120, non_cooperative=nc, progress={'window': 10})
    split, whole = out['progress_partials_split'], out['progress_partials']
    counts = [0, 1, 2, 3, 4, 7, 8, 9, 10, 11, 14, 15, 16]
    assert np.array_equal(split[:, :, counts].sum(1), whole[:, counts])
    assert np.allclose(split.sum(1), whole, rtol=1e-12)
    assert np.array_equal(split[:, :, 7:10].sum(2), out['partials_split'][:, :, 3])
    assert out['progress_by_role']['non_cooperative']['unfinished'] == int(split[:, 1, 7:10].sum())


def test_evaluate_cli_timeouts_json(built, tmp_path, capsys):
    import evaluate
    path = tmp_path / 'progress.json'
    argv = ['--scenario', 'stage2', '--policy', os.path.join(CKPT, 'stage1_2.pth'), '--num-worlds', '4', '--episodes',
            '1', '--json', str(path)]
    evaluate.main(argv)
    plain_bytes = path.read_bytes()
    plain = json.loads(plain_bytes)
    assert 'progress' not in plain and 'timeouts' not in plain['args'] and 'stall_window' not in plain['args']
    plain_lines = capsys.readouterr().out.strip().splitlines()
    evaluate.main(argv + ['--timeouts'])
    first = path.read_bytes()
    evaluate.main(argv + ['--timeouts'])
    assert path.read_bytes() == first
    lines = capsys.readouterr().out.strip().splitlines()
    assert lines[0] == plain_lines[0] and lines[1].startswith('progress  time-outs ')
    d = json.loads(first)
    assert d['partials'] == plain['partials'] and d['ticks'] == plain['ticks']
    assert d['progress']['params']['window'] == 50 and np.asarray(d['progress']['partials']).shape == (4, 19)
    m = d['progress']['metrics']
    assert m['timeouts'] == d['metrics']['timed_out'] and m['unfinished'] == d['metrics']['unfinished']
    evaluate.main(argv + ['--stall-window', '10'])
    d10 = json.loads(path.read_bytes())
    assert d10['progress']['params']['window'] == 10
    assert d10['progress']['metrics']['timeouts'] == m['timeouts']
    # without the flags the output is what it was
    evaluate.main(argv)
    assert path.read_bytes() == plain_bytes
