"""Training on a mix of scenarios on the device (DESIGN.md §9l): composing env handles on column slices of one rollout
changes no component, a one-component mix is the single-env run, and trainer.run / ppo_stage2.py --mix end to end."""
import logging
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
NAMES = ('stage2', 'random', 'circle')


def _envs(seed=0, names=NAMES):
    """Stage 2 (4 worlds), random K = 8 (16 worlds, 6 m square, 25-tick time-out) and a circle of 8 robots on a 3 m
    circle (4 worlds), each built as a single-scenario run builds it."""
    from rl_collision_avoidance_b200.circle_world import StageWorld as CircleWorld
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from rl_collision_avoidance_b200.stage_world2 import StageWorld as Stage2World
    make = {'stage2': lambda: Stage2World(512, num_worlds=4, seed=seed, auto_reset=2),
            'random': lambda: StageWorld(512, scenario=make_scenario('random', robots_per_world=8, side=6.0, timeout=25),
                                         num_worlds=16, seed=seed, auto_reset=0),
            'circle': lambda: CircleWorld(512, num_env=8, radius=3.0, num_worlds=4, seed=seed, auto_reset=2)}
    return [make[n]() for n in names]


def _tsame(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _steer(gs, noise):
    """Full speed with the heading error turned at gain 2, plus noise (as tests/test_relayout_gpu.py drives)."""
    w = torch.clamp(2.0 * torch.atan2(gs[:, 1], gs[:, 0]) + noise[:, 1], -1.0, 1.0)
    return torch.stack((torch.clamp(1.0 - noise[:, 0].abs(), 0.0, 1.0), w), 1).contiguous()


def test_composition_changes_no_component(built):
    """The mix and one standalone env per scenario, each through trainer.compose / start / tick, driven by the same
    action bits (seeded noise around goal seeking; not the policy, whose last bits may depend on the batch size).
    After every horizon each component's slice of stacks, gs, rewards, flags and eplog, its state, live mask and
    re-layout status equal its standalone env's bit for bit; group re-spawns and re-layouts happen."""
    from rl_collision_avoidance_b200.trainer import Rollout, compose
    H, horizons = 80, 3                                  # 240 ticks: past stage 2's 200-tick time-out
    mix = _envs(seed=3)
    alone = _envs(seed=3)
    N = sum(e.N for e in mix)
    ro = Rollout(H, N, 512, 'cuda')
    comps = compose(mix, ro)
    solo = [(compose([e], r)[0], r) for e, r in ((e, Rollout(H, e.N, 512, 'cuda')) for e in alone)]
    for c in comps + [s for s, _ in solo]:
        c.start()
    gen = torch.Generator(device='cuda').manual_seed(11)
    reset_seen = {n: 0 for n in NAMES}
    for h in range(horizons):
        for t in range(H):
            ro.scaled.copy_(_steer(ro.gs[t], 0.5 * torch.randn(N, 2, device='cuda', generator=gen)))
            for c, (s, r) in zip(comps, solo):
                r.scaled.copy_(ro.scaled[c.a:c.b])
                c.tick(t)
                s.tick(t)
        torch.cuda.synchronize()
        for c, (s, r) in zip(comps, solo):
            n = c.name
            for key in ('stacks', 'gs', 'rewards', 'flags', 'eplog'):
                assert _tsame(getattr(c, key), getattr(r, key)), f'horizon {h}: {n} {key}'
            for key in ('pose', 'goal', 'acc', 'meta'):
                assert _tsame(c.env.state[key], s.env.state[key]), f'horizon {h}: {n} state {key}'
            if c.relayout:
                assert _tsame(c.env.live, s.env.live), f'horizon {h}: {n} live'
                assert _tsame(c.env._relayout_status, s.env._relayout_status), f'horizon {h}: {n} status'
                c.env.check_relayout()
            reset_seen[n] += int(c.flags[:, :, 3].sum())
        ro.stacks[0].copy_(ro.stacks[H])
        ro.gs[0].copy_(ro.gs[H])
        for s, r in solo:
            r.stacks[0].copy_(r.stacks[H])
            r.gs[0].copy_(r.gs[H])
    assert all(v > 0 for v in reset_seen.values()), reset_seen           # group re-spawns and re-layouts happened
    rnd = comps[NAMES.index('random')].env
    assert int(rnd.state['meta'][:, 1].max()) >= 3                       # some world past its second re-layout


class ListHandler(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def _train(tmp_path, updates, envs, seed=1, tag='a', save_every=3):
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.trainer import run
    n = sum(e.N for e in envs) if isinstance(envs, list) else envs.N
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(128, n))
    policy.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    before = policy.flat.clone()
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=64, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=128, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=44, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    lg = logging.getLogger(f'test_mix_{tag}')
    lg.setLevel(logging.INFO)
    h = ListHandler()
    lg.addHandler(h)
    gen = torch.Generator(device='cuda').manual_seed(seed)
    stats = run(env=envs, policy=policy, policy_path=str(tmp_path), action_bound=[[0, -1], [1, 1]], optimizer=opt,
                hp=hp, logger=lg, logger_cal=None, stage=2, max_updates=updates, save_every=save_every, generator=gen)
    lg.removeHandler(h)
    return policy, before, stats, h.lines


@pytest.mark.parametrize('name', ['stage2', 'random'])
def test_one_component_mix_is_the_single_env_run(built, tmp_path, name):
    e1, = _envs(seed=4, names=(name,))
    e2, = _envs(seed=4, names=(name,))
    a = _train(tmp_path / 'a', 2, e1, seed=4, tag='one_a', save_every=100)
    b = _train(tmp_path / 'b', 2, [e2], seed=4, tag='one_b', save_every=100)
    assert _tsame(a[0].flat, b[0].flat)
    assert a[3] == b[3]                                             # the same log lines, byte for byte
    for k in ('pose', 'goal', 'acc', 'meta'):
        assert _tsame(e1.state[k], e2.state[k]), k
    assert [s['by_scenario'] for s in a[2]] == [s['by_scenario'] for s in b[2]]


@pytest.mark.parametrize('name', ['stage2', 'random'])
def test_single_env_run_equals_the_trainer_before_mixes(built, name):
    """run(env) against tests/golden/trainer_single_env.json, recorded with the trainer before mixed runs existed:
    the same parameters, state and Env log lines bit for bit, and the same per-update stats."""
    import json
    from trainer_golden import GOLDEN, record
    from rl_collision_avoidance_b200.trainer import run
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = record(run, name)
    for key in ('params', 'state', 'log', 'log_lines'):
        assert got[key] == want[key], key
    assert json.dumps(got['stats'], sort_keys=True) == json.dumps(want['stats'], sort_keys=True)
    assert got['log_lines'] > 0


def test_trainer_runs_on_a_mix(built, tmp_path):
    envs = _envs(seed=1)
    policy, before, stats, lines = _train(tmp_path, 3, envs)
    assert len(stats) == 3 and all(np.isfinite(s['losses']).all() for s in stats)
    assert float((policy.flat - before).abs().max()) > 0 and torch.isfinite(policy.flat).all()
    env_lines = [l for l in lines if l.startswith('Env ')]
    for e in envs:
        mine = [l for l in env_lines if l.endswith(', ' + e.sc.name)]
        assert mine, (e.sc.name, env_lines[:5])
        robots = {int(l.split(',')[0][4:]) for l in mine}
        assert max(robots) < e.num_env                              # indexed within the component's own world
    assert all(any(l.endswith(', ' + n) for n in NAMES) for l in env_lines)
    for s in stats:
        assert set(s['by_scenario']) == set(NAMES)
        assert sum(v['episodes'] for v in s['by_scenario'].values()) == s['episodes']
        assert s['agent_steps_per_s'] > 0
    assert sum(s['by_scenario'][n]['episodes'] for s in stats for n in NAMES) == len(env_lines)
    assert all(sum(s['by_scenario'][n]['episodes'] for s in stats) > 0 for n in NAMES)
    path = tmp_path / 'stage2_3.pth'
    assert path.exists() and (tmp_path / 'stage2_3.pth.trainer').exists()
    import evaluate
    out = evaluate.main(['--scenario', 'stage2', '--policy', str(path), '--num-worlds', '2'])
    assert out['metrics']['episodes'] > 0


def test_mixed_training_is_deterministic(built, tmp_path):
    ea, eb = _envs(seed=5), _envs(seed=5)
    a = _train(tmp_path / 'a', 2, ea, seed=5, tag='d1', save_every=100)
    b = _train(tmp_path / 'b', 2, eb, seed=5, tag='d2', save_every=100)
    assert _tsame(a[0].flat, b[0].flat)
    for x, y in zip(ea, eb):
        for k in ('pose', 'goal', 'acc', 'meta'):
            assert _tsame(x.state[k], y.state[k]), (x.sc.name, k)


def test_trainer_rejects_a_bad_mix(built):
    from rl_collision_avoidance_b200.circle_world import StageWorld as CircleWorld
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.stage_world1 import StageWorld as Stage1World
    from rl_collision_avoidance_b200.stage_world2 import StageWorld as Stage2World
    from rl_collision_avoidance_b200.trainer import run
    pol = CNNPolicy(seed=0, max_batch=512)
    opt = Adam(pol.parameters(), lr=5e-5)
    go = lambda envs, stage=2: run(env=envs, policy=pol, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt,
                                   hp=dict(HORIZON=4), stage=stage, max_updates=1)
    s2, rnd, cir = _envs(names=NAMES)
    with pytest.raises(ValueError, match='a mix of scenarios trains with stage 2, got stage 1'):
        go([s2, cir], stage=1)
    with pytest.raises(ValueError, match='stage 1 cannot be mixed'):
        go([s2, Stage1World(512, num_worlds=1, auto_reset=1)])
    with pytest.raises(ValueError, match='stage2 appears more than once'):
        go([s2, cir, Stage2World(512, num_worlds=1, auto_reset=2)])
    with pytest.raises(ValueError, match='circle trains with auto_reset 2 in a mix, got 0'):
        go([s2, CircleWorld(512, num_env=8, radius=3.0, num_worlds=1, auto_reset=0)])
    with pytest.raises(ValueError, match='share the device and the beam count'):
        go([s2, CircleWorld(256, num_env=8, radius=3.0, num_worlds=1, auto_reset=2)])
    with pytest.raises(ValueError, match='stage 2 and auto_reset 0'):
        go([rnd, cir], stage=1)


def test_ppo_stage2_mix_end_to_end(built, tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'ppo_stage2.py'), '--mix', 'stage2:2,random:8,circle:1',
                        '--random-robots', '8', '--updates', '2', '--policy-path', str(tmp_path / 'policy')],
                       cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert 'update 2:' in r.stdout, r.stdout[-2000:]
    for name, cols in (('stage2', '[0, 88)'), ('random', '[88, 152)'), ('circle', '[152, 202)')):
        assert ('  %s: ' % name) in r.stdout and ('columns %s' % cols) in r.stdout, r.stdout[-2000:]
    assert any(l.endswith(', random') for l in r.stdout.splitlines() if l.startswith('Env '))
