"""Safety metrics on the device (csrc/rlca_safety.cu, DESIGN.md §9m): rlca_safety_track against its host twin bit for
bit on every scenario and episode mechanic, the clearance against torch.amin, consistency with the episode tracker,
evaluate() with the option on against the recorded partials, determinism and shard invariance, causes on free floor,
the split by role, and evaluate.py --safety end to end."""
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
INF = np.float32(np.inf)


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cpu'))
    return pol


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _host_state(N, E):
    return dict(min_sep=np.full(N, INF, np.float32), min_clear=np.full(N, INF, np.float32),
                last_clear=np.full(N, INF, np.float32), near=np.zeros(N, np.int32),
                partner=np.full(N, -1, np.int32), records=np.zeros((N, E, 4), np.float32))


def _np(t):
    return t.cpu().numpy()


# (id, scenario keywords, auto_reset, worlds, beams, near_dist, expects re-spawns, misaligned scan buffer)
TRACK_CASES = [
    ('stage1', dict(name='stage1'), 1, 2, 512, 0.3, True, False),
    ('stage2', dict(name='stage2'), 2, 2, 512, 0.3, True, False),
    ('circle16', dict(name='circle', robots_per_world=16, radius=4.0), 0, 2, 512, 0.3, False, False),
    ('random2', dict(name='random', robots_per_world=2, side=3.0, separation=0.8, min_travel=1.5), 0, 6, 512, 0.3,
     False, False),
    ('random8', dict(name='random', robots_per_world=8, side=5.0, separation=0.8, min_travel=2.0), 0, 3, 512, 0.3,
     False, False),
    ('random64', dict(name='random', robots_per_world=64, side=14.0, separation=0.8, min_travel=5.0), 0, 1, 512, 0.3,
     False, False),
    ('one_robot_510_beams', dict(name='stage1', robots_per_world=1), 1, 32, 510, 0.3, True, False),
    ('misaligned_scan', dict(name='stage1'), 1, 1, 512, 0.3, True, True),
]


@pytest.mark.parametrize('case', TRACK_CASES, ids=[c[0] for c in TRACK_CASES])
def test_device_track_equals_host_twin(built, case):
    """300 random-action ticks: running state and records of the kernel equal rlca_safety_track_host fed with the same
    poses, flags, scans and tracker state; the clearance equals torch.amin of the tick's scan in metres."""
    from rl_collision_avoidance_b200.evaluation import EpisodeTracker, SafetyTracker, safety_track_host
    from rl_collision_avoidance_b200.stage_world import StageWorld
    _, kw, auto_reset, worlds, beams, near, respawns, misaligned = case
    kw = dict(kw)
    sc = make_scenario(kw.pop('name'), **kw)
    env = StageWorld(beams, scenario=sc, num_worlds=worlds, seed=21, auto_reset=auto_reset)
    env.reset_pose()
    if sc.layout is not None:
        env.random_layout()
    E = 3
    tr = EpisodeTracker(env, E)
    st = SafetyTracker(env, tr, near)
    host = _host_state(env.N, E)
    shifted = None
    if misaligned:                                                 # a copy of the scans whose rows start 4 bytes off 16
        shifted = torch.zeros(env.N * beams + 1, device='cuda')[1:].view(env.N, beams)
        assert shifted.data_ptr() % 16 == 4
    rng = np.random.default_rng(22)
    seen_respawn = seen_crash = 0
    for t in range(300):
        a = random_actions(rng, env.N)
        pose_in, meta_in = _np(env.state['pose']), _np(env.state['meta'])
        env.control_vel(torch.from_numpy(a).cuda())
        closed, count = _np(tr.closed), _np(tr.count)
        if misaligned:
            shifted.copy_(env.obs)
            _track_with_io(env, st, tr, env._io(action=env._keep[0], obs=shifted))
        else:
            st.track()
        tr.track()
        obs = shifted if misaligned else env.obs
        flags = _np(env.flags)
        safety_track_host(env.cfg, near, pose_in, meta_in, _np(env.state['pose']), flags, _np(obs), closed, count, host)
        seen_respawn += int(flags[:, 3].sum())
        seen_crash += int((flags[:, 2] == 2).sum())
        if t % 50 == 49 or t < 3:
            for k in host:
                assert _bits_equal(_np(getattr(st, k)), host[k]), (t, k)
            want = (torch.amin(obs, 1) + 0.5) * float(env.cfg.range_max)
            assert torch.equal(st.last_clear, want), t
    rec, cnt = host['records'], np.minimum(_np(tr.count), E)
    assert cnt.sum() > 0 or sc.robots_per_world == 2
    assert seen_crash > 0 or sc.robots_per_world == 2 or misaligned
    assert (seen_respawn > 0) == respawns
    if sc.robots_per_world >= 8:
        assert any((rec[a, :cnt[a], 2] > 0).any() for a in range(env.N)), 'no near-miss tick in the run'
    # consistency with the tracker: a cause exactly where its result is Crashed
    res = _np(tr.records)
    for a in range(env.N):
        cause = rec[a, :cnt[a], 3].astype(np.int64) & 3
        assert np.array_equal(cause != 0, res[a, :cnt[a], 0] == 2), a
        assert not rec[a, cnt[a]:].any()
    if sc.layout is not None:                                      # free floor: nothing static to hit
        assert all(((rec[a, :cnt[a], 3].astype(np.int64) & 3) != 1).all() for a in range(env.N))
    if sc.robots_per_world == 1:
        assert all(((rec[a, :cnt[a], 3].astype(np.int64) & 3) != 2).all() for a in range(env.N))


def _track_with_io(env, st, tr, io):
    import ctypes as C
    from rl_collision_avoidance_b200 import _lib
    s_in, s_out = env._state_struct(1 - env._cur), env._state_struct(env._cur)
    _lib.check(env.lib.rlca_safety_track(C.byref(env.cfg), C.byref(st._params), C.byref(s_in), C.byref(s_out),
                                         C.byref(io), C.byref(tr._st), C.byref(st._st), env._stream()))


def _golden_run(name, safety):
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController, OrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    scenario, worlds, seed, who, episodes, max_ticks, check_every = make_golden_eval.RUNS[name]
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])
    policy = OrcaController(env) if who == 'orca' else NhOrcaController(env, obstacles=True) if who == 'nh-orca' \
        else _policy(who, env.N)
    return env, evaluate(env, policy, episodes, max_ticks, check_every=check_every, safety=safety)


def test_evaluate_with_safety_keeps_the_recorded_partials(built):
    """Every run of tests/golden/eval_partials.npz with the option on: the same partials and ticks bit for bit, the
    device reduction equal to the host reduction, and the causes consistent with the crash column."""
    from rl_collision_avoidance_b200.evaluation import SAFETY_COLUMNS, safety_reduce_host
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_partials.npz'))
    for name in make_golden_eval.RUNS:
        env, out = _golden_run(name, 0.1)
        assert out['ticks'] == int(g['ticks_' + name]), name
        assert np.array_equal(out['partials'].view(np.uint64), g['partials_' + name].view(np.uint64)), name
        sp, tr, st = out['safety_partials'], out['tracker'], out['safety_tracker']
        assert sp.shape == (env.num_worlds, len(SAFETY_COLUMNS))
        host = safety_reduce_host(env.cfg, _np(st.records), _np(tr.records), _np(tr.count))
        assert _bits_equal(sp, host), name
        assert np.array_equal(sp[:, 0] + sp[:, 1], out['partials'][:, 1]), name      # static + robot = crashed
        assert np.array_equal(sp[:, 4], out['partials'][:, 0]), name                 # reached
        assert (sp[:, 2] <= sp[:, 1]).all() and not sp[:, 3].any()
    _, plain = _golden_run('stage2_policy', None)
    assert not any(k.startswith('safety') for k in plain)


def test_safety_is_deterministic_and_shard_invariant(built):
    from rl_collision_avoidance_b200.evaluation import evaluate, safety_totals
    from rl_collision_avoidance_b200.orca import NhOrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('random', robots_per_world=8, side=6.0, separation=0.8, min_travel=3.0)

    def run(W, off, safety=0.1):
        env = StageWorld(512, scenario=sc, num_worlds=W, seed=5, auto_reset=0, world_offset=off)
        return evaluate(env, NhOrcaController(env, obstacles=True), 1, 300, safety=safety)

    a, b = run(8, 0), run(8, 0)
    assert _bits_equal(a['safety_partials'], b['safety_partials']) and _bits_equal(a['partials'], b['partials'])
    parts = np.concatenate([run(4, off)['safety_partials'] for off in (0, 4)])
    assert _bits_equal(parts, a['safety_partials'])
    assert _bits_equal(safety_totals(parts), a['safety_totals'])
    assert a['safety_totals'][4] > 0 and np.isfinite(a['safety']['min_separation'])
    assert not a['safety_partials'][:, 0].any()                   # free floor: no static crash
    plain = run(8, 0, None)
    assert _bits_equal(plain['partials'], a['partials']) and plain['ticks'] == a['ticks']


def test_random_policy_crashes_are_robot_crashes_and_roles_add_up(built):
    """stage2.pth on packed random layouts and on the circle with non-cooperative robots: no static cause on free floor;
    the two roles' partials add up to the unsplit ones; crashes into a non-cooperative robot are robot crashes."""
    from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask
    from rl_collision_avoidance_b200.orca import NonCooperative
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('random', robots_per_world=16, side=6.0, separation=0.8, min_travel=3.0)
    env = StageWorld(512, scenario=sc, num_worlds=8, seed=1, auto_reset=0)
    out = evaluate(env, _policy('stage2.pth', env.N), 1, 300, safety=0.1)
    tot = out['safety_totals']
    assert tot[0] == 0 and tot[1] == out['totals'][1] and tot[1] > 0
    sc = make_scenario('circle', robots_per_world=12, radius=4.0)
    env = StageWorld(512, scenario=sc, num_worlds=6, seed=2, auto_reset=0)
    nc = NonCooperative(env, non_cooperative_mask(12, 6, 2))
    out = evaluate(env, _policy('stage2.pth', env.N), 1, 300, non_cooperative=nc, safety=0.1)
    split, whole = out['safety_partials_split'], out['safety_partials']
    counts = [0, 1, 2, 4, 5, 8, 11, 12]
    assert np.array_equal(split[:, :, counts].sum(1), whole[:, counts])
    assert np.allclose(split[:, :, [6, 7, 9, 10]].sum(1), whole[:, [6, 7, 9, 10]], rtol=1e-12)
    assert np.array_equal(split[:, :, 13].min(1), whole[:, 13])
    assert (split[:, 0, 3] <= split[:, 0, 1]).all() and (split[:, 1, 3] <= split[:, 1, 1]).all()
    assert out['safety_by_role']['cooperative']['crash_into_masked'] == int(split[:, 0, 3].sum())
    assert split[:, :, 1].sum() > 0


def test_evaluate_cli_safety_json(built, tmp_path, capsys):
    import evaluate
    path = tmp_path / 'safety.json'
    argv = ['--scenario', 'stage2', '--policy', os.path.join(CKPT, 'stage2.pth'), '--num-worlds', '4', '--episodes', '1',
            '--json', str(path)]
    evaluate.main(argv)
    plain = json.loads(path.read_bytes())
    assert 'safety' not in plain and 'safety' not in plain['args'] and 'near_miss' not in plain['args']
    plain_lines = capsys.readouterr().out.strip().splitlines()
    evaluate.main(argv + ['--safety'])
    first = path.read_bytes()
    evaluate.main(argv + ['--safety'])
    assert path.read_bytes() == first
    lines = capsys.readouterr().out.strip().splitlines()
    assert lines[0] == plain_lines[0] and lines[1].startswith('safety  crashes static ')
    d = json.loads(first)
    assert d['partials'] == plain['partials'] and d['ticks'] == plain['ticks']
    assert d['safety']['near_miss'] == 0.1 and np.asarray(d['safety']['partials']).shape == (4, 14)
    m = d['safety']['metrics']
    assert m['crash_static'] + m['crash_robot'] == d['metrics']['crashed'] and m['reached'] == d['metrics']['reached']
    evaluate.main(argv + ['--near-miss', '0.5'])
    assert json.loads(path.read_bytes())['safety']['metrics']['near_episodes'] >= m['near_episodes']
