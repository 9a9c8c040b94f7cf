"""Training on random layouts on the device (DESIGN.md §9k): rlca_layout_respawn against its host twin after every
tick, the refreshed scan stacks and goal | speed rows, the env after a re-layout against the CPU oracle, determinism and
sharding of whole rollouts, and trainer.run / ppo_stage2.py --scenario random end to end."""
import logging
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, random_actions

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _env(K, W, timeout, seed=0, world_offset=0, S=10.0):
    """A random-scenario env with auto_reset 0 right after its first layout, as trainer.run starts it."""
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('random', robots_per_world=K, side=S, timeout=timeout)
    env = StageWorld(512, scenario=sc, num_worlds=W, seed=seed, auto_reset=0, world_offset=world_offset)
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    env.random_layout()
    return env


class Driver:
    """The trainer's per-tick sequence with seeded random actions: tick with `live` into the stack / gs / flags
    buffers, then relayout_finished."""

    def __init__(self, env, horizon):
        n, dev = env.N, env.device
        self.env, self.H = env, horizon
        self.stacks = torch.empty(horizon + 1, n, 3, 512, device=dev)
        self.gs = torch.empty(horizon + 1, n, 4, device=dev)
        self.flags = torch.zeros(horizon, n, 4, dtype=torch.uint8, device=dev)
        self.eplog = torch.zeros(horizon, n, 8, device=dev)
        self.rewards = torch.zeros(horizon, n, device=dev)
        self.stacks[0] = env.obs[:, None, :]
        self.gs[0] = env.gs

    def tick(self, t, action):
        e = self.env
        e.control_vel(action, live=e.live, stack_in=self.stacks[t], stack_out=self.stacks[t + 1],
                      out={'reward': self.rewards[t], 'flags': self.flags[t], 'gs': self.gs[t + 1],
                           'eplog': self.eplog[t]})

    def relayout(self, t):
        self.env.relayout_finished(self.stacks[t + 1], out={'gs': self.gs[t + 1], 'flags': self.flags[t]})

    def carry(self):
        self.stacks[0].copy_(self.stacks[self.H])
        self.gs[0].copy_(self.gs[self.H])


def _host(env, flags):
    torch.cuda.synchronize()
    st = env.state
    return (st['pose'].cpu().numpy(), st['goal'].cpu().numpy(), st['acc'].cpu().numpy(), st['meta'].cpu().numpy(),
            flags.cpu().numpy())


def _same(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8),
                                                 np.ascontiguousarray(b).view(np.uint8))


def _tsame(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _steer(gs, noise):
    """Full speed with the heading error turned at gain 2, plus noise: robots reach goals and collide at different
    ticks, so worlds end their episodes at different ticks."""
    w = torch.clamp(2.0 * torch.atan2(gs[:, 1], gs[:, 0]) + noise[:, 1], -1.0, 1.0)
    return torch.stack((torch.clamp(1.0 - noise[:, 0].abs(), 0.0, 1.0), w), 1).contiguous()


@pytest.mark.parametrize('K,W,S,timeout,T', [(4, 1024, 6.0, 60, 130), (8, 256, 6.0, 60, 130),
                                             (32, 1024, 10.0, 25, 90)])
def test_device_equals_host_after_every_tick(built, K, W, S, timeout, T):
    """T ticks of noisy goal-seeking actions with `live`: after every tick the state, live, status and flags equal the
    host twin applied to the tick's output; re-laid rows of the stack and gs are the new scan and local goal, every
    other row keeps the tick's bits; every world is re-laid at least twice, and with K <= 8 not all at the same
    ticks."""
    from rl_collision_avoidance_b200.scenarios import relayout_host
    env = _env(K, W, timeout=timeout, seed=K, S=S)
    d = Driver(env, T)
    gen = torch.Generator(device='cuda').manual_seed(K)
    relaid_count = np.zeros(W, np.int64)
    first_relaid = np.full(W, -1)
    for t in range(T):
        d.tick(t, _steer(d.gs[t], 0.5 * torch.randn(env.N, 2, device='cuda', generator=gen)))
        before = _host(env, d.flags[t])
        stack_tick, gs_tick = d.stacks[t + 1].clone(), d.gs[t + 1].clone()
        d.relayout(t)
        want = relayout_host(env.cfg, env.sc.layout, *before)
        got = _host(env, d.flags[t]) + (env.live.cpu().numpy(), env._relayout_status.cpu().numpy())
        for name, x, y in zip(('pose', 'goal', 'acc', 'meta', 'flags', 'live', 'status'), got, want):
            assert _same(x, y), f'tick {t}: {name} differs'
        assert not want[6].any()
        relaid = torch.from_numpy(want[4][:, 3] != 0).cuda()
        r = d.stacks[t + 1][relaid]
        assert _tsame(r, env.obs[relaid][:, None, :].expand(-1, 3, -1)), f'tick {t}: refreshed stack'
        assert _tsame(d.gs[t + 1][relaid], env.gs[relaid]), f'tick {t}: refreshed gs'
        assert _tsame(d.stacks[t + 1][~relaid], stack_tick[~relaid]), f'tick {t}: other stack rows'
        assert _tsame(d.gs[t + 1][~relaid], gs_tick[~relaid]), f'tick {t}: other gs rows'
        per_world = want[4][:, 3].reshape(W, K).all(1)
        relaid_count += per_world
        first_relaid[(first_relaid < 0) & per_world] = t
    # the refreshed scans are the lidar's from the new poses
    assert _tsame(env.raycast(env.state['pose'], normalise=True), env.obs)
    assert relaid_count.min() >= 2, relaid_count.min()
    if K <= 8:              # a world of 32 robots rarely ends every episode before a 25-tick time-out
        assert len(np.unique(first_relaid)) > 1


def test_oracle_parity_after_relayout(built):
    """After the first re-layout of a 16-world env, the oracle with the same state and live mask: scan and local goal
    equal, then 20 random-action ticks stay bit-exact in state, scan, local goal and flags."""
    from oracle.oracle import OracleWorld, OrcConfig
    from rl_collision_avoidance_b200.scenarios import fill_config
    K, W = 8, 16
    env = _env(K, W, timeout=15, seed=7)
    d = Driver(env, 40)
    rng = np.random.default_rng(7)
    for t in range(40):
        d.tick(t, torch.from_numpy(random_actions(rng, env.N)).cuda())
        d.relayout(t)
        if bool(d.flags[t][:, 3].any()):
            break
    else:
        raise AssertionError('no world was re-laid in 40 ticks')
    ocfg = fill_config(OrcConfig(), env.sc, num_worlds=W, beams=512, auto_reset=0, seed=7)
    orc = OracleWorld(ocfg, env.sc.map.cells, env.sc.init_tab, env.sc.goal_tab)
    torch.cuda.synchronize()
    for k in ('pose', 'goal', 'acc', 'meta'):
        getattr(orc, k)[...] = env.state[k].cpu().numpy()
    orc.observe()
    assert_outputs_equal(env, orc, 'relayout')
    live = env.live.clone()
    for t in range(20):
        a = random_actions(rng, orc.N)
        env.control_vel(torch.from_numpy(a).cuda(), live=live)
        orc.step(a, live=live.cpu().numpy())
        assert_state_equal(env, orc, f'tick {t}')
        assert_outputs_equal(env, orc, f'tick {t}')
        assert np.array_equal(env.flags.cpu().numpy(), orc.flags), f'tick {t}: flags differ'


def _rollout(K, W, seed, world_offset=0, horizons=3, H=30, actions=None):
    env = _env(K, W, timeout=20, seed=seed, world_offset=world_offset)
    d = Driver(env, H)
    out = {k: [] for k in ('stacks', 'flags', 'eplog', 'gs', 'pose', 'meta')}
    for h in range(horizons):
        for t in range(H):
            a = actions[h * H + t][world_offset * K:(world_offset + W) * K]
            d.tick(t, torch.from_numpy(np.ascontiguousarray(a)).cuda())
            d.relayout(t)
        torch.cuda.synchronize()
        env.check_relayout()
        out['stacks'].append(d.stacks.cpu().numpy())
        out['flags'].append(d.flags.cpu().numpy())
        out['eplog'].append(d.eplog.cpu().numpy())
        out['gs'].append(d.gs.cpu().numpy())
        out['pose'].append(env.state['pose'].cpu().numpy())
        out['meta'].append(env.state['meta'].cpu().numpy())
        d.carry()
    return {k: np.stack(v) for k, v in out.items()}


def test_rollouts_are_deterministic_and_shard_invariant(built):
    K, W, H, horizons = 8, 20, 30, 3
    rng = np.random.default_rng(3)
    actions = [random_actions(rng, K * W) for _ in range(H * horizons)]
    a = _rollout(K, W, 5, actions=actions)
    b = _rollout(K, W, 5, actions=actions)
    for k in a:
        assert _same(a[k], b[k]), k
    assert (a['meta'][-1][:, 1] >= 3).any()                     # some world is past its second re-layout
    parts = [_rollout(K, wc, 5, world_offset=w0, actions=actions) for w0, wc in ((0, 12), (12, 8))]
    for k in a:
        axis = 1 if k in ('pose', 'meta') else 2                 # the agent axis
        assert _same(np.concatenate([p[k] for p in parts], axis=axis), a[k]), k


class ListHandler(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def _train(tmp_path, updates, seed=1, tag='a', save_every=3):
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.trainer import run
    env = _env(8, 16, timeout=40, seed=seed)
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(128, env.N))
    policy.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    before = policy.flat.clone()
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=64, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=128, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=8, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    lg = logging.getLogger(f'test_relayout_{tag}')
    lg.setLevel(logging.INFO)
    h = ListHandler()
    lg.addHandler(h)
    gen = torch.Generator(device='cuda').manual_seed(seed)
    stats = run(env=env, policy=policy, policy_path=str(tmp_path), action_bound=[[0, -1], [1, 1]], optimizer=opt,
                hp=hp, logger=lg, logger_cal=None, stage=2, max_updates=updates, save_every=save_every, generator=gen)
    lg.removeHandler(h)
    return env, policy, before, stats, h.lines


def test_trainer_runs_on_random_layouts(built, tmp_path, capsys):
    env, policy, before, stats, lines = _train(tmp_path, 3)
    assert len(stats) == 3 and all(np.isfinite(s['losses']).all() for s in stats)
    assert float((policy.flat - before).abs().max()) > 0 and torch.isfinite(policy.flat).all()
    env_lines = [l for l in lines if l.startswith('Env ')]
    assert env_lines and all('Goal (' in l and l.endswith(',') for l in env_lines), env_lines[:3]
    assert int(env.state['meta'][:, 1].max()) >= 3
    path = tmp_path / 'stage2_3.pth'
    assert path.exists() and (tmp_path / 'stage2_3.pth.trainer').exists()
    import evaluate
    out = evaluate.main(['--scenario', 'random', '--policy', str(path), '--num-worlds', '4'])
    assert out['metrics']['episodes'] > 0


def test_trainer_rejects_random_without_stage2_and_auto_reset0(built, tmp_path):
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from rl_collision_avoidance_b200.trainer import run
    for stage, auto_reset in ((1, 0), (2, 2)):
        env = StageWorld(512, scenario=make_scenario('random'), num_worlds=2, auto_reset=auto_reset)
        pol = CNNPolicy(seed=0, max_batch=env.N)
        with pytest.raises(ValueError, match='stage 2 and auto_reset 0'):
            run(env=env, policy=pol, policy_path=None, action_bound=[[0, -1], [1, 1]],
                optimizer=Adam(pol.parameters(), lr=5e-5), hp=dict(HORIZON=4), stage=stage, max_updates=1)


def test_training_is_deterministic(built, tmp_path):
    a = _train(tmp_path / 'a', 2, seed=4, tag='d1', save_every=100)
    b = _train(tmp_path / 'b', 2, seed=4, tag='d2', save_every=100)
    assert _tsame(a[1].flat, b[1].flat)
    for k in ('pose', 'goal', 'acc', 'meta'):
        assert _tsame(a[0].state[k], b[0].state[k]), k


def test_ppo_stage2_random_end_to_end(built, tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'ppo_stage2.py'), '--scenario', 'random', '--random-robots',
                        '8', '--num-worlds', '8', '--updates', '2', '--policy-path', str(tmp_path / 'policy')],
                       cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert 'update 2:' in r.stdout, r.stdout[-2000:]
