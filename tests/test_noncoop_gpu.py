"""Non-cooperative robots on the device (DESIGN.md §9h): rlca_noncoop_action against its host twin, the split
reduction after evaluate(), the action override inside the tick loop, the circle rule, evaluate() without the feature
against the partials recorded before it existed, and evaluate.py end to end."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from helpers import random_actions

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cpu'))
    return pol


def _env(scenario, worlds, seed, sc=None):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.stage_world import StageWorld
    return StageWorld(512, scenario=sc or scenario, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])


def _host_state(env):
    st = env.state
    return st['pose'].cpu().numpy(), st['goal'].cpu().numpy(), st['meta'].cpu().numpy()


def _masks(env, rng):
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    R, W = env.cfg.robots_per_world, env.num_worlds
    return {'none': np.zeros(env.N, np.uint8), 'all': np.ones(env.N, np.uint8),
            'spaced': non_cooperative_mask(R, W, min(5, R)),
            'random': (rng.random(env.N) < 0.4).astype(np.uint8) * rng.integers(1, 256, env.N).astype(np.uint8)}


@pytest.mark.parametrize('scenario,worlds', [('stage1', 171), ('stage2', 8), ('circle', 4)])
def test_driver_matches_host_twin(built, scenario, worlds):
    from rl_collision_avoidance_b200.orca import NonCooperative, noncoop_host
    env = _env(scenario, worlds, seed=21)
    env.reset_pose()
    rng = np.random.default_rng(21)
    for _ in range(25):
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda())
    pose, goal, meta = _host_state(env)
    for name, mask in _masks(env, rng).items():
        for speed, gain in ((None, 2.0), (0.55, 0.8)):
            act0 = rng.uniform(-3, 3, (env.N, 2)).astype(np.float32)
            act0[::11, 1] = np.nan
            act = torch.from_numpy(act0).cuda()
            NonCooperative(env, mask, speed=speed, heading_gain=gain).apply(act)
            got = act.cpu().numpy()
            want = noncoop_host(env.cfg, pose, goal, meta, mask, act0, speed=speed, heading_gain=gain)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, speed)
            keep = mask == 0
            assert np.array_equal(got[keep].view(np.uint32), act0[keep].view(np.uint32)), name
            if mask.any():
                assert not np.array_equal(got[~keep].view(np.uint32), act0[~keep].view(np.uint32)), name


def test_split_partials_match_host_reduction(built):
    from rl_collision_avoidance_b200.evaluation import (evaluate, metrics, non_cooperative_mask, reduce_split_host,
                                                        totals)
    from rl_collision_avoidance_b200.orca import NonCooperative
    env = _env('stage2', 3, seed=2)
    nc = NonCooperative(env, non_cooperative_mask(env.cfg.robots_per_world, 3, 5))
    out = evaluate(env, _policy('stage2.pth', env.N), 2, max_ticks=402, non_cooperative=nc)
    tr = out['tracker']
    host = reduce_split_host(env.cfg, tr.records.cpu().numpy(), tr.count.cpu().numpy(), tr.open.cpu().numpy(),
                             nc.mask.cpu().numpy())
    split = out['partials_split']
    assert split.shape == (3, 2, 14)
    assert np.array_equal(host.view(np.uint64), split.view(np.uint64))
    assert np.array_equal(split[:, 0, :4] + split[:, 1, :4], out['partials'][:, :4])
    assert np.array_equal(tr.partials_split(nc.mask, 1, 2), split[1:3])
    by = out['by_role']
    assert by['non_cooperative']['episodes'] > 0 and by['cooperative']['episodes'] > 0
    for role, row in (('cooperative', 0), ('non_cooperative', 1)):
        want = metrics(totals(split[:, row]))
        assert all(by[role][k] == want[k] for k in ('episodes', 'reached', 'crashed', 'timed_out', 'unfinished'))


def test_override_reaches_the_tick(built):
    """A hand-driven NH-ORCA loop on stage 2: the action control_vel receives for every masked agent is the host
    driver's action from the state before the tick; the others keep the controller's."""
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    from rl_collision_avoidance_b200.orca import NhOrcaController, NonCooperative, noncoop_host
    env = _env('stage2', 4, seed=8)
    env.reset_pose()
    ctrl = NhOrcaController(env)
    mask = non_cooperative_mask(env.cfg.robots_per_world, 4, 3)
    nc = NonCooperative(env, mask, speed=0.8)
    for t in range(60):
        pose, goal, meta = _host_state(env)
        raw = ctrl()
        before = raw.cpu().numpy()
        env.control_vel(nc.apply(raw))
        sent = env._keep[0].cpu().numpy()
        want = noncoop_host(env.cfg, pose, goal, meta, mask, before, speed=0.8)
        assert np.array_equal(sent.view(np.uint32), want.view(np.uint32)), t


def test_circle_rule_stops_terminated_non_cooperative_robots(built):
    """Inside evaluate() on a 12-robot circle: a non-cooperative robot gets its driver's action until it terminates;
    from the next tick on its v is 0 although the driver would move it."""
    from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask
    from rl_collision_avoidance_b200.orca import NonCooperative, noncoop_host
    from rl_collision_avoidance_b200.scenarios import make_scenario
    env = _env('circle', 1, seed=6, sc=make_scenario('circle', robots_per_world=12, radius=6.0))
    mask = non_cooperative_mask(12, 1, 3)
    log = []
    step = env.control_vel

    def control_vel(action, **kw):
        pose, goal, meta = _host_state(env)
        sent = action.cpu().numpy()
        step(action, **kw)
        log.append((pose, goal, meta, sent, env.flags[:, 0].cpu().numpy() != 0))

    env.control_vel = control_vel
    evaluate(env, _policy('stage2.pth', env.N), 1, max_ticks=240, check_every=240,
             non_cooperative=NonCooperative(env, mask))
    env.control_vel = step
    stopped = driven = 0
    terminal = np.zeros(env.N, bool)
    for pose, goal, meta, sent, done in log:
        drv = noncoop_host(env.cfg, pose, goal, meta, mask, sent)
        for a in np.flatnonzero(mask):
            if terminal[a]:
                assert sent[a, 0] == 0.0 and sent[a, 1:].view(np.uint32) == drv[a, 1:].view(np.uint32), a
                stopped += int(drv[a, 0] > 0)
            else:
                assert np.array_equal(sent[a].view(np.uint32), drv[a].view(np.uint32)), a
                driven += 1
        terminal = done
    assert stopped > 0 and driven > 0, (stopped, driven)


def _golden_run(name, zero_mask=False):
    """A run of tools/make_golden_eval.RUNS, optionally with a NonCooperative whose mask is all zero."""
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController, NonCooperative, OrcaController
    scenario, worlds, seed, who, episodes, max_ticks, check_every = make_golden_eval.RUNS[name]
    env = _env(scenario, worlds, seed)
    if who == 'orca':
        policy = OrcaController(env)
    elif who == 'nh-orca':
        policy = NhOrcaController(env, obstacles=True)
    else:
        policy = _policy(who, env.N)
    nc = NonCooperative(env, np.zeros(env.N, np.uint8)) if zero_mask else None
    return evaluate(env, policy, episodes, max_ticks, check_every=check_every, non_cooperative=nc)


def test_evaluate_without_the_feature_keeps_its_partials(built):
    """evaluate() without non_cooperative: the per-world partials and tick counts recorded before the feature existed
    (tests/golden/eval_partials.npz, tools/make_golden_eval.py), bit for bit."""
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_partials.npz'))
    for name in make_golden_eval.RUNS:
        out = _golden_run(name)
        assert 'by_role' not in out and 'partials_split' not in out
        assert out['ticks'] == int(g['ticks_' + name]), name
        assert np.array_equal(out['partials'].view(np.uint64), g['partials_' + name].view(np.uint64)), name


@pytest.mark.parametrize('name', ['stage1_policy', 'circle_orca'])
def test_all_zero_mask_changes_nothing(built, name):
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_partials.npz'))
    out = _golden_run(name, zero_mask=True)
    assert np.array_equal(out['partials'].view(np.uint64), g['partials_' + name].view(np.uint64))
    assert np.array_equal(out['partials_split'][:, 0].view(np.uint64), out['partials'].view(np.uint64))
    assert not out['partials_split'][:, 1].any()


def test_evaluate_cli_json_is_deterministic(built, tmp_path, capsys):
    import evaluate
    path = tmp_path / 'noncoop.json'
    argv = ['--scenario', 'stage1', '--policy', os.path.join(CKPT, 'stage1_2.pth'), '--num-worlds', '2',
            '--episodes', '2', '--max-ticks', '200', '--non-cooperative', '5', '--json', str(path)]
    evaluate.main(argv)
    first = path.read_bytes()
    evaluate.main(argv)
    assert path.read_bytes() == first
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 6 and 'non-cooperative  stage1  robots 10' in lines[-1]
    d = json.loads(first)
    assert np.asarray(d['partials_split']).shape == (2, 2, 14)
    split = np.asarray(d['partials_split'])
    assert np.array_equal(split[:, 0, :4] + split[:, 1, :4], np.asarray(d['partials'])[:, :4])
    assert d['by_role']['non_cooperative']['episodes'] > 0


def test_head_on_non_cooperative_pair_crashes(built, capsys):
    """K = 2 on a 4 m circle, both non-cooperative: they meet head-on on the diameter and both first records are
    crashes."""
    import evaluate
    out = evaluate.main(['--scenario', 'circle', '--circle-robots', '2', '--circle-radius', '4', '--baseline', 'orca',
                         '--non-cooperative', '2', '--max-ticks', '120', '--check-every', '10'])
    tr = out['tracker']
    assert list(tr.count.cpu().numpy()) == [1, 1]
    assert list(tr.records.cpu().numpy()[:, 0, 0]) == [2.0, 2.0]
    assert out['by_role']['non_cooperative']['crashed'] == 2 and out['by_role']['cooperative']['episodes'] == 0
