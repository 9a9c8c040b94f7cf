"""Training with the global planner on the device (DESIGN.md §9x): rlca_plan_shape against its host twin bit for bit at
the evaluation shapes, in place and out of place, and after every tick of rollouts with re-spawns and re-layouts;
inside trainer.run, ro.gs and ro.rewards against the field, waypoint and shaping twins on the recorded states; the
'straight' arm's rewards; and deterministic training."""
import numpy as np
import pytest
import torch

from helpers import random_actions

pytestmark = pytest.mark.gpu


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _np(t):
    return t.detach().cpu().numpy().copy()


def _scenario(name, K=16, T=64, timeout=None):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    if name == 'arena':
        return make_scenario('arena', robots_per_world=K, arenas=T, pick=1, timeout=timeout)
    return make_scenario(name)


AUTO_RESET = {'stage1': 1, 'stage2': 2, 'arena': 0}


class _Twin:
    """The host twins of one Planner(reward=True), carried along with the device planner."""

    def __init__(self, planner):
        from rl_collision_avoidance_b200.planner import HostState
        self.p, self.env = planner, planner.env
        self.hs = HostState(self.env.cfg, planner.tables)
        self.pp = np.zeros(self.env.N, np.float32)
        self.ps = np.zeros(self.env.N, np.float32)

    def step(self, pose, goal, gs_in, flags=None, reward=None, eplog=None):
        """Twin outputs (gs, reward, eplog) on host copies of the inputs."""
        from rl_collision_avoidance_b200.planner import fields_host, shape_host
        env = self.env
        fields_host(env.cfg, self.p.tables, self.hs, goal)
        gs = np.array(gs_in, np.float32, copy=True)
        reward = None if reward is None else np.array(reward, np.float32, copy=True)
        eplog = None if eplog is None else np.array(eplog, np.float32, copy=True)
        shape_host(env.cfg, self.p.tables, self.hs, self.pp, self.ps, pose, goal, gs, flags, reward, eplog,
                   in_place=True)
        return gs, reward, eplog

    def check(self):
        p = self.p
        assert _same(_np(p.psi_prev), self.pp) and _same(_np(p.psi_start), self.ps)
        assert _same(_np(p.status()), self.hs.status) and _same(_np(p.status_count), self.hs.status_count)
        assert _same(_np(p.entry), self.hs.entry)


@pytest.mark.parametrize('name, W, ticks', [('stage1', 171, 3), ('stage2', 24, 3), ('arena', 1024, 3),
                                            ('stage1', 8, 200), ('stage2', 2, 300), ('arena', 16, 250)])
def test_shape_kernel_equals_twin(built, name, W, ticks):
    """The first update out of place (gs_in env.gs, gs_out the planner's buffer), then one per tick in place on copies
    of the tick's gs, reward and eplog, every output against the twin bit for bit."""
    from rl_collision_avoidance_b200.planner import Planner
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = _scenario(name)
    env = StageWorld(512, scenario=sc, num_worlds=W, seed=3, auto_reset=AUTO_RESET[name])
    env.reset_world()
    env.reset_pose()
    if sc.layout is not None:
        env.random_layout()
    planner = Planner(env, reward=True)
    tw = _Twin(planner)
    st = env.state
    gs_twin, _, _ = tw.step(_np(st['pose']), _np(st['goal']), _np(env.gs))
    out = planner.update(None)
    torch.cuda.synchronize()
    assert out is planner.gs and _same(_np(out), gs_twin)
    tw.check()
    rng = np.random.default_rng(0)
    ro_gs = torch.empty(env.N, 4, device='cuda')
    ro_rw = torch.empty(env.N, device='cuda')
    ro_ep = torch.zeros(env.N, 8, device='cuda')
    flags = torch.zeros(env.N, 4, dtype=torch.uint8, device='cuda')
    seen = np.zeros(4, np.int64)
    for t in range(ticks):
        a = random_actions(rng, env.N)
        a[:, 0] = np.abs(a[:, 0])
        env.control_vel(torch.from_numpy(a).cuda(), live=env.live if sc.layout is not None else None,
                        out={'gs': ro_gs, 'reward': ro_rw, 'eplog': ro_ep, 'flags': flags})
        if sc.layout is not None:
            env.relayout_finished(torch.empty(env.N, 3, 512, device='cuda'), out={'gs': ro_gs, 'flags': flags})
        torch.cuda.synchronize()
        st = env.state
        fl = _np(flags)
        gs_twin, rw_twin, ep_twin = tw.step(_np(st['pose']), _np(st['goal']), _np(ro_gs), fl, _np(ro_rw), _np(ro_ep))
        planner.update(flags, reward=ro_rw, eplog=ro_ep, gs=ro_gs)
        torch.cuda.synchronize()
        assert _same(_np(ro_gs), gs_twin) and _same(_np(ro_rw), rw_twin) and _same(_np(ro_ep), ep_twin), t
        tw.check()
        seen += [(fl[:, 0] == 0).sum(), (fl[:, 2] != 0).sum(), (fl[:, 3] != 0).sum(), (_np(planner.status()) == 1).sum()]
    if ticks > 10:
        assert seen.min() > 0, seen                   # shaped ticks, episode ends, re-spawns / re-layouts, waypoints


def _recorder(monkeypatch):
    """Record what trainer.run's ticks leave, for the twins: wrap StageWorld.control_vel and relayout_finished (the
    reward, eplog, gs and flags the tick and the re-layout wrote, before any planner), _Component.start and
    _Component.tick (the env state each leaves), and capture the Rollout.  Returns (records, rollouts)."""
    from rl_collision_avoidance_b200 import trainer
    from rl_collision_avoidance_b200.stage_world import StageWorld
    recs, rollouts, raw = [], [], {}
    cv, rf = StageWorld.control_vel, StageWorld.relayout_finished
    start, tick, Rollout = trainer._Component.start, trainer._Component.tick, trainer.Rollout

    def control_vel(self, action, live=None, obs_out=None, stack_in=None, stack_out=None, out=None):
        cv(self, action, live=live, obs_out=obs_out, stack_in=stack_in, stack_out=stack_out, out=out)
        torch.cuda.synchronize()
        raw[id(self)] = {k: _np(out[k]) for k in ('reward', 'eplog', 'gs', 'flags')}

    def relayout_finished(self, stack_out, out=None):
        rf(self, stack_out, out=out)
        torch.cuda.synchronize()
        raw[id(self)].update(gs=_np(out['gs']), flags=_np(out['flags']))

    def state(c):
        torch.cuda.synchronize()
        return dict(comp=c, pose=_np(c.env.state['pose']), goal=_np(c.env.state['goal']))

    def start_(self):
        start(self)
        r = state(self)
        r.update(gs=_np(self.env.gs), gs_slot=_np(self.gs[0]))      # env.gs: what slot 0 held before the planner
        recs.append(r)

    def tick_(self, t):
        tick(self, t)
        r = state(self)
        r.update(t=t, **raw[id(self.env)])
        recs.append(r)

    class _Rollout(Rollout):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            rollouts.append(self)
    monkeypatch.setattr(StageWorld, 'control_vel', control_vel)
    monkeypatch.setattr(StageWorld, 'relayout_finished', relayout_finished)
    monkeypatch.setattr(trainer._Component, 'start', start_)
    monkeypatch.setattr(trainer._Component, 'tick', tick_)
    monkeypatch.setattr(trainer, 'Rollout', _Rollout)
    return recs, rollouts


def _train(envs, seed, planner, updates=2, horizon=32, noise=None, latency=None):
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.trainer import run
    N = sum(e.N for e in envs)
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(128, N))
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=horizon, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=128, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=envs[0].cfg.robots_per_world, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    stats = run(env=envs if len(envs) > 1 else envs[0], policy=policy, policy_path=None,
                action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp, stage=1 if envs[0].sc.name == 'stage1' else 2,
                max_updates=updates, generator=torch.Generator(device='cuda').manual_seed(seed), noise=noise,
                latency=latency, planner=planner)
    return policy, stats


def _envs(kind, seed):
    from rl_collision_avoidance_b200.stage_world import StageWorld
    if kind == 'stage1':
        return [StageWorld(512, scenario=_scenario('stage1'), num_worlds=4, seed=seed, auto_reset=1)]
    if kind == 'arena':
        return [StageWorld(512, scenario=_scenario('arena', 8, 16, 40), num_worlds=16, seed=seed, auto_reset=0)]
    return [StageWorld(512, scenario=_scenario('stage2'), num_worlds=1, seed=seed, auto_reset=2),
            StageWorld(512, scenario=_scenario('arena', 8, 16, 40), num_worlds=16, seed=seed, auto_reset=0)]


def _check_rollout(recs, ro, H, shape=True):
    """The twins run on every recorded state against the rollout slots PPO reads: ro.gs[0] after the start (before
    the horizon's carry overwrote it, so its snapshot), ro.gs[t + 1], ro.rewards[t] and ro.eplog[t] after tick t.
    Without `shape` the rewards and eplog must be the tick's.  Returns (shaped rewards, episode ends)."""
    twins = {}
    gs_all, rw_all, ep_all = _np(ro.gs), _np(ro.rewards), _np(ro.eplog)
    shaped = ends = 0
    for r in recs:
        c = r['comp']
        tw = twins.setdefault(id(c), _Twin(c.planner))
        if 't' not in r:
            gs, _, _ = tw.step(r['pose'], r['goal'], r['gs'])
            assert _same(r['gs_slot'], gs)
            continue
        t, cols = r['t'], slice(c.a, c.b)
        gs, rw, ep = tw.step(r['pose'], r['goal'], r['gs'], r['flags'], r['reward'], r['eplog'])
        assert _same(gs_all[t + 1, cols], gs), t
        if shape:
            assert _same(rw_all[t, cols], rw) and _same(ep_all[t, cols], ep), t
        else:
            assert _same(rw_all[t, cols], r['reward']) and _same(ep_all[t, cols], r['eplog']), t
        shaped += int((rw_all[t, cols] != r['reward']).sum())
        ends += int(((r['flags'][:, 0] != 0) & (r['flags'][:, 2] != 0)).sum())
    assert len([r for r in recs if 't' in r]) == len(twins) * H
    return shaped, ends


@pytest.mark.parametrize('kind', ['stage1', 'arena', 'mix'])
def test_trainer_rollout_equals_twins(built, monkeypatch, kind):
    """One update of trainer.run with planner='geodesic' (noise and latency on in the stage 2 + arena mix): the rollout
    slots PPO reads, ro.gs[t + 1], ro.rewards[t] and ro.eplog[t], equal the field, waypoint and shaping twins run on
    the state each tick left, with the reward, eplog, gs and flags the tick and the re-layout wrote."""
    from rl_collision_avoidance_b200.latency import LatencyParams
    from rl_collision_avoidance_b200.noise import NoiseParams
    recs, rollouts = _recorder(monkeypatch)
    extra = dict(noise=NoiseParams(range_sigma=0.02, dropout=0.05, v_gain_sigma=0.05, w_gain_sigma=0.05, seed=1),
                 latency=LatencyParams(scan_delay=(0, 2), command_delay=(0, 1), seed=2)) if kind == 'mix' else {}
    _, stats = _train(_envs(kind, 6), 6, 'geodesic', updates=1, horizon=48, **extra)
    assert 'planner' in stats[-1] and stats[-1]['planner']['robot_ticks'] > 0
    assert len(rollouts) == 1
    shaped, ends = _check_rollout(recs, rollouts[0], 48)
    assert shaped > 0 and ends > 0


def test_straight_keeps_the_tick_reward(built, monkeypatch):
    """planner='straight': ro.gs holds the waypoints and ro.rewards / ro.eplog exactly what the tick wrote for the
    same state and command, which is the reward an unplanned tick gives."""
    recs, rollouts = _recorder(monkeypatch)
    _train(_envs('arena', 7), 7, 'straight', updates=1, horizon=48)
    assert all(r['comp'].planner.reward is False for r in recs)
    _check_rollout(recs, rollouts[0], 48, shape=False)
    steered = sum(int((r['gs'] != _np(rollouts[0].gs[r['t'] + 1, r['comp'].a:r['comp'].b])).any(1).sum())
                  for r in recs if 't' in r)
    assert steered > 0


def test_training_with_the_planner_is_deterministic(built):
    a_pol, a = _train(_envs('mix', 8), 8, 'geodesic')
    b_pol, b = _train(_envs('mix', 8), 8, 'geodesic')
    assert torch.equal(a_pol.flat, b_pol.flat)
    for x, y in zip(a, b):
        for k in ('episodes', 'mean_ep_reward', 'success_rate', 'losses', 'by_scenario', 'planner'):
            assert repr(x[k]) == repr(y[k]), k


def test_ppo_stage2_arena_with_planner_trains(built, tmp_path):
    """ppo_stage2.py --scenario arena --planner end to end, from stage2.pth in a scratch directory."""
    import os
    import shutil
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    (tmp_path / 'policy').mkdir()
    shutil.copy(os.path.join(root, 'tests', 'golden', 'checkpoints', 'stage2.pth'), tmp_path / 'policy' / 'stage2.pth')
    out = subprocess.run([sys.executable, os.path.join(root, 'ppo_stage2.py'), '--scenario', 'arena', '--arena-robots',
                          '8', '--arena-count', '8', '--arena-timeout', '60', '--num-worlds', '16', '--updates', '2',
                          '--planner'], cwd=tmp_path, capture_output=True, text=True, check=True).stdout
    assert 'update 2:' in out and 'last update, planner: goal_visible' in out, out[-2000:]
