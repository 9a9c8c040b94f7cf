"""The hybrid controller on the device (DESIGN.md §9j): rlca_hybrid_action against its host twin on every scenario, the
counters against per-tick snapshots, evaluate() with the hybrid disabled against the partials recorded before it
existed, determinism and sharding with the defaults, the composition with non-cooperative robots, and evaluate.py end
to end."""
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
F = np.float32


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cpu'))
    return pol


def _env(scenario, worlds, seed, world_offset=0):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('random', robots_per_world=8) if scenario == 'random' else scenario
    return StageWorld(512, scenario=sc, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario],
                      world_offset=world_offset)


def _host_state(env):
    torch.cuda.synchronize()
    st = env.state
    return st['pose'].cpu().numpy(), st['goal'].cpu().numpy(), st['meta'].cpu().numpy()


def _bits(a):
    return np.asarray(a).view(np.uint32)


def _distance(cfg, stack):
    return (stack[:, 2].min(1) + F(0.5)) * F(cfg.range_max)


def _ticked(scenario, worlds, seed, ticks=25):
    """An env after `ticks` random-action ticks through a scan FIFO, as evaluate() resets it, and the FIFO the next
    tick reads."""
    env = _env(scenario, worlds, seed)
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    if env.sc.layout is not None:
        env.random_layout()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, env.beam_mum, device='cuda')]
    rng = np.random.default_rng(seed)
    for t in range(ticks):
        k = t & 1
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda(), stack_in=stacks[k],
                        stack_out=stacks[1 - k])
    return env, stacks[ticks & 1]


@pytest.mark.parametrize('scenario,worlds', [('stage1', 171), ('stage2', 8), ('circle', 4), ('random', 1024)])
def test_device_equals_host_twin(built, scenario, worlds):
    """Action, mode and counts bit for bit, at the 1/3 and 2/3 quantiles of d (every mode occurs) and at the
    defaults, from random actions laced with NaN, random open flags and nonzero counters."""
    from rl_collision_avoidance_b200.evaluation import EpisodeTracker
    from rl_collision_avoidance_b200.orca import HYBRID_DEFAULTS, Hybrid, hybrid_host
    env, stack = _ticked(scenario, worlds, seed=21)
    pose, goal, meta = _host_state(env)
    st = stack.cpu().numpy()
    d = _distance(env.cfg, st)
    lo, hi = (float(np.quantile(d, q, method='lower')) for q in (1 / 3, 2 / 3))
    rng = np.random.default_rng(worlds)
    tracker = EpisodeTracker(env, 1)
    open_ = (rng.random(env.N) < 0.7).astype(np.int32)
    tracker.open.copy_(torch.from_numpy(open_))
    for prm in (dict(r_safe=hi, r_risk=lo), dict(r_safe=hi, r_risk=lo, v_safe=0.3, heading_gain=1.2),
                dict(HYBRID_DEFAULTS)):
        hy = Hybrid(env, **prm)
        counts0 = rng.integers(0, 100, (env.N, 3)).astype(np.int32)
        hy.counts.copy_(torch.from_numpy(counts0))
        act0 = rng.uniform(-3, 3, (env.N, 2)).astype(np.float32)
        act0[::11, 0] = np.nan
        act = torch.from_numpy(act0).cuda()
        hy.apply(act, stack, tracker)
        want = hybrid_host(env.cfg, st, pose, goal, meta, act0, open_, counts0, **prm)
        assert np.array_equal(_bits(act.cpu().numpy()), _bits(want[0])), prm
        assert np.array_equal(hy.mode.cpu().numpy(), want[1]), prm
        assert np.array_equal(hy.counts.cpu().numpy(), want[2]), prm
        if prm['r_safe'] == hi:
            assert all((want[1] == k).any() for k in range(3)), np.bincount(want[1])
        # without a tracker nothing is counted
        hy.apply(torch.from_numpy(act0).cuda(), stack)
        assert np.array_equal(hy.counts.cpu().numpy(), want[2])


def test_counts_are_the_sum_of_per_tick_modes(built):
    """A hand-driven stage2.pth loop on stage 2 with the defaults: counts = sum over ticks of one-hot(mode) * open,
    with open snapshotted before each tick."""
    from rl_collision_avoidance_b200.evaluation import ACTION_BOUND, EpisodeTracker
    from rl_collision_avoidance_b200.model.ppo import generate_action_no_sampling
    from rl_collision_avoidance_b200.orca import Hybrid
    env = _env('stage2', 3, seed=5)
    env.reset_pose()
    pol = _policy('stage2.pth', env.N)
    tracker = EpisodeTracker(env, 1)
    tracker.reset()
    hy = Hybrid(env)
    hy.reset()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, env.beam_mum, device='cuda')]
    want = np.zeros((env.N, 3), np.int64)
    for t in range(300):
        k = t & 1
        _, scaled = generate_action_no_sampling(env=env, state_list=(stacks[k], env.get_local_goal(),
                                                                     env.get_self_speed()),
                                                policy=pol, action_bound=ACTION_BOUND)
        open_ = tracker.open.cpu().numpy()
        hy.apply(scaled, stacks[k], tracker)
        want += np.eye(3, dtype=np.int64)[hy.mode.cpu().numpy()] * (open_ != 0)[:, None]
        env.control_vel(scaled, stack_in=stacks[k], stack_out=stacks[1 - k])
        tracker.track()
    got = hy.counts.cpu().numpy()
    assert np.array_equal(got, want)
    assert (want.sum(0) > 0).all(), want.sum(0)
    assert np.array_equal(hy.counts_per_world(), want.reshape(3, -1, 3).sum(1))


def _golden_run(name, hybrid=None):
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import Hybrid
    scenario, worlds, seed, who, episodes, max_ticks, check_every = make_golden_eval.RUNS[name]
    env = _env(scenario, worlds, seed)
    hy = None if hybrid is None else Hybrid(env, **hybrid(env))
    return evaluate(env, _policy(who, env.N), episodes, max_ticks, check_every=check_every, hybrid=hy)


def test_disabled_hybrid_reproduces_the_golden_partials(built):
    """r_risk = 0 and r_safe = range_max: the policy runs of tests/golden/eval_partials.npz bit for bit, and every
    counted tick is mode 0."""
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_partials.npz'))
    off = lambda env: dict(r_safe=float(env.cfg.range_max), r_risk=0.0)
    names = [n for n, run in make_golden_eval.RUNS.items() if run[3].endswith('.pth')]
    assert len(names) == 3
    for name in names:
        out = _golden_run(name, off)
        assert out['ticks'] == int(g['ticks_' + name]), name
        assert np.array_equal(out['partials'].view(np.uint64), g['partials_' + name].view(np.uint64)), name
        mc = out['mode_counts']
        assert mc.dtype == np.int64 and mc.shape == (out['partials'].shape[0], 3)
        assert mc[:, 0].sum() > 0 and not mc[:, 1:].any(), name
        assert out['modes']['policy'] == 1.0 and out['modes']['agent_ticks'] == mc.sum()


def _random_eval(W, seed, world_offset=0, nc=None, max_ticks=300):
    from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask
    from rl_collision_avoidance_b200.orca import Hybrid, NonCooperative
    env = _env('random', W, seed, world_offset)
    ncc = None if nc is None else NonCooperative(env, non_cooperative_mask(8, W, nc))
    hy = Hybrid(env)
    # one completion check at the end: every shard runs the same ticks
    return env, hy, evaluate(env, _policy('stage2.pth', env.N), 1, max_ticks, check_every=max_ticks,
                             non_cooperative=ncc, hybrid=hy)


def test_defaults_are_deterministic_and_shard_invariant(built):
    _, _, a = _random_eval(24, 3)
    _, _, b = _random_eval(24, 3)
    assert a['ticks'] == b['ticks']
    assert np.array_equal(a['partials'].view(np.uint64), b['partials'].view(np.uint64))
    assert np.array_equal(a['mode_counts'], b['mode_counts'])
    mc = a['mode_counts']
    assert (mc.sum(0) > 0).all(), mc.sum(0)              # every mode occurs with the defaults
    parts = [_random_eval(wc, 3, world_offset=w0)[2] for w0, wc in ((0, 16), (16, 8))]
    assert [p['ticks'] for p in parts] == [a['ticks']] * 2
    assert np.array_equal(np.concatenate([p['partials'] for p in parts]).view(np.uint64),
                          a['partials'].view(np.uint64))
    assert np.array_equal(np.concatenate([p['mode_counts'] for p in parts]), mc)


def test_composes_with_non_cooperative_robots(built):
    """--non-cooperative 2 on random with the hybrid: until a masked robot terminates, the action its tick receives is
    the driver's from the pre-tick state; the mode counts cover the cooperative robots only."""
    from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask
    from rl_collision_avoidance_b200.orca import Hybrid, NonCooperative, mode_shares, noncoop_host
    W = 8
    env = _env('random', W, 2)
    mask = non_cooperative_mask(8, W, 2)
    log = []
    step = env.control_vel

    def control_vel(action, **kw):
        pose, goal, meta = _host_state(env)
        sent = action.cpu().numpy()
        step(action, **kw)
        log.append((pose, goal, meta, sent, env.flags[:, 0].cpu().numpy() != 0))

    env.control_vel = control_vel
    hy = Hybrid(env)
    out = evaluate(env, _policy('stage2.pth', env.N), 1, 200, check_every=200,
                   non_cooperative=NonCooperative(env, mask), hybrid=hy)
    env.control_vel = step
    terminal = np.zeros(env.N, bool)
    driven = 0
    for pose, goal, meta, sent, done in log:
        drv = noncoop_host(env.cfg, pose, goal, meta, mask, sent)
        live = (mask != 0) & ~terminal
        assert np.array_equal(_bits(sent[live]), _bits(drv[live]))
        driven += int(live.sum())
        terminal = done
    assert driven > 0
    everyone = hy.counts_per_world()
    coop = hy.counts_per_world(mask)
    assert np.array_equal(out['mode_counts'], coop)
    assert (everyone - coop).sum() > 0                    # the masked robots were counted, and left out
    assert out['modes'] == mode_shares(coop)
    assert set(out['by_role']) == {'cooperative', 'non_cooperative'}


def test_evaluate_cli_json_is_deterministic(built, tmp_path, capsys):
    import evaluate
    path = tmp_path / 'hybrid.json'
    argv = ['--scenario', 'random', '--policy', os.path.join(CKPT, 'stage2.pth'), '--num-worlds', '16', '--hybrid',
            '--json', str(path)]
    evaluate.main(argv)
    first = path.read_bytes()
    evaluate.main(argv)
    assert path.read_bytes() == first
    d = json.loads(first)
    assert np.asarray(d['mode_counts']).shape == (16, 3)
    assert d['modes']['agent_ticks'] == np.asarray(d['mode_counts']).sum()
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 4 and lines[1].startswith('hybrid modes over ')
