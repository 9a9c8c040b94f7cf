"""Acceleration limits on the device (DESIGN.md §9r): the kernel against the host twin bit for bit over 20-tick
sequences with resets and crashes at the bench shape and at R = 1, 44 and 64; stage 1 end to end, tick by tick (no
speed step above limit dt, the env's own buffers untouched, re-spawns at the rate of a run without limits);
evaluate() with non-binding limits bit-identical to a run without, with binding limits deterministic, and together
with noise, latency and NH-ORCA; rollouts with the FIFO invariants and PPO updates under limits on stage 1, on random
layouts with re-layouts and on a mix."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from test_latency_gpu import _bits, _check_fifo, _cfg, _policy, _tsame

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
BOTH = dict(linear=(1.0, 1.0), angular=(2.0, 2.0), seed=3)
RANGED = dict(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=2 ** 40 + 17)
LOOSE = dict(linear=(10.0, 10.0), angular=(20.0, 20.0), seed=5)


def _action_device(cfg, p, bufs, draw, flags, cmd, out, stream_id):
    from rl_collision_avoidance_b200 import _lib
    st = _lib.DynamicsState(*(b.data_ptr() for b in bufs))
    fp = C.c_void_p(flags.data_ptr()) if flags is not None else None
    _lib.check(_lib.load().rlca_dynamics_action(C.byref(cfg), C.byref(p.struct(stream_id)), C.byref(st), draw, fp,
                                                C.c_void_p(cmd.data_ptr()), C.c_void_p(out.data_ptr()), None))


@pytest.mark.parametrize('R,W,offset', [(24, 171, 0), (1, 300, 5), (44, 12, 3), (64, 9, 0), (24, 10, 2)])
def test_kernel_equals_host_twin(built, R, W, offset):
    """20 ticks: the first call without flags, then random resets and crashes (or, for one setting, no flags at all:
    every row fresh on every call); commands in and out of the bounds, with NaN, +-inf and -0"""
    from rl_collision_avoidance_b200.dynamics import DynamicsParams, HostState, action_host
    from test_dynamics import _commands
    cfg = _cfg(R, W, 8, world_offset=offset * 10)
    N = R * W
    rng = np.random.default_rng(R * 1000 + offset)
    for k, (p, with_flags) in enumerate(((DynamicsParams(**RANGED), True), (DynamicsParams(**BOTH), True),
                                         (DynamicsParams(linear=(0.5, 0.5), seed=1), True),
                                         (DynamicsParams(angular=(3.0, 3.0), seed=2), True),
                                         (DynamicsParams(**RANGED), False))):
        hs = HostState(cfg)
        bufs = (torch.zeros(N, 2, device='cuda'), torch.zeros(N, device='cuda'), torch.zeros(N, device='cuda'))
        out = torch.empty(N, 2, device='cuda')
        prev = None
        for t in range(20):
            cmd = _commands(rng, N)
            cin = torch.from_numpy(cmd).cuda()
            ex = action_host(cfg, p, hs, t, cmd, prev, stream_id=k)
            _action_device(cfg, p, bufs, t, None if prev is None else torch.from_numpy(prev).cuda(), cin, out, k)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(out), _bits(ex)), (k, t)
            assert np.array_equal(_bits(cin), _bits(cmd))
            assert np.array_equal(_bits(bufs[0]), _bits(hs.vel)), (k, t)
            assert np.array_equal(_bits(bufs[1]), _bits(hs.lin_limit)), (k, t)
            assert np.array_equal(_bits(bufs[2]), _bits(hs.ang_limit)), (k, t)
            if with_flags:
                prev = np.zeros((N, 4), np.uint8)
                prev[rng.random(N) < 0.1, 3] = 1
                prev[rng.random(N) < 0.1, 1] = 1


def _stage1(kw, ticks, seed=1):
    """stage 1 driven by stage1_2.pth's mean action plus noise, tick by tick, with limits `kw` (None: without); per
    tick the step checks; returns the (ticks, N) bool re-spawn flags"""
    from rl_collision_avoidance_b200.dynamics import Dynamics, DynamicsParams
    from rl_collision_avoidance_b200.model.ppo import generate_action_no_sampling
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=seed, auto_reset=1)
    dyn = None if kw is None else Dynamics(env, DynamicsParams(**kw))
    pol = _policy('stage1_2.pth', env.N)
    gen = torch.Generator(device='cuda').manual_seed(seed)
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, 512, device='cuda')]
    resets = []
    for tick in range(ticks):
        k = tick & 1
        _, scaled = generate_action_no_sampling(env=env, state_list=(stacks[k], env.get_local_goal(),
                                                                     env.get_self_speed()),
                                                policy=pol, action_bound=[[0, -1], [1, 1]])
        scaled = scaled + 0.3 * torch.randn(scaled.shape, device='cuda', generator=gen)
        cmd = scaled
        if dyn is not None:
            prev = env.flags.clone() if tick > 0 else None
            speed = env.gs[:, 2:4].clone()
            issued = scaled.clone()
            snap = {'obs': env.obs.clone(), 'gs': env.gs.clone(), 'flags': env.flags.clone()}
            snap.update({'state_' + n: t.clone() for n, t in env.state.items()})
            cmd = dyn.action(scaled, prev)
            torch.cuda.synchronize()
            assert _tsame(scaled, issued)
            for n in ('obs', 'gs', 'flags'):
                assert _tsame(getattr(env, n), snap[n]), (tick, n)
            for n, t in env.state.items():
                assert _tsame(t, snap['state_' + n]), (tick, n)
        env.control_vel(cmd, stack_in=stacks[k], stack_out=stacks[1 - k])
        torch.cuda.synchronize()
        fresh_now = env.flags[:, 3] != 0
        resets.append(fresh_now.cpu().numpy())
        if dyn is not None:
            # the speed the tick drove with is the executed command (rows it did not re-spawn), and it moved from the
            # speed of the tick before by at most limit dt, for rows that neither started an episode nor crashed
            keep = ~fresh_now
            assert torch.equal(env.gs[keep, 2:4], cmd[keep]), tick
            if prev is not None:
                live = keep & (prev[:, 3] == 0) & (prev[:, 1] == 0)
                step = (env.gs[:, 2:4].double() - speed.double()).abs()
                lim = (dyn.limits * float(env.cfg.dt)).double()         # limit dt rounded to float32, as applied
                slack = torch.maximum(env.gs[:, 2:4].abs(), speed.abs()).double() * 2.0 ** -24
                assert bool((step[live] <= lim[live] + slack[live]).all()), tick
    return np.stack(resets)


def test_stage1_end_to_end_tick_by_tick(built):
    """Stage 1 re-spawns inside the tick.  A re-spawned robot starts from rest, so it must still move on its first
    tick: re-spawns per tick stay at the rate of the same run without limits (a robot held still after a crash would
    crash again on every tick)"""
    with_limits, without = _stage1(RANGED, 120), _stage1(None, 120)
    n = with_limits.shape[1]
    per_tick = lambda f: f.sum(1).tolist()
    again = lambda f: int((f[1:] & f[:-1]).sum())          # re-spawned on two ticks in a row
    assert with_limits.sum() > 0 and without.sum() > 0
    assert with_limits.sum() <= 3 * without.sum() + n // 2, (per_tick(with_limits), per_tick(without))
    assert again(with_limits) <= 2 * again(without) + n // 8, (per_tick(with_limits), per_tick(without))


def _evaluate(dyn_kw, noise_kw=None, latency_kw=None, scenario='stage1', worlds=6, ticks=80, seed=3, baseline=None):
    from rl_collision_avoidance_b200.dynamics import Dynamics, DynamicsParams
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate
    from rl_collision_avoidance_b200.latency import Latency, LatencyParams
    from rl_collision_avoidance_b200.noise import Noise, NoiseParams
    from rl_collision_avoidance_b200.orca import NhOrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])
    dyn = None if dyn_kw is None else Dynamics(env, DynamicsParams(**dyn_kw))
    lat = None if latency_kw is None else Latency(env, LatencyParams(**latency_kw))
    noise = None if noise_kw is None else Noise(env, NoiseParams(**noise_kw))
    pol = NhOrcaController(env) if baseline else _policy('stage1_2.pth', env.N)
    before = env.launch_count
    out = evaluate(env, pol, 2, ticks, check_every=20, safety=0.1, noise=noise, latency=lat, dynamics=dyn)
    torch.cuda.synchronize()
    return env, out, env.launch_count - before


def _same_run(a, b):
    ea, oa, la = a
    eb, ob, lb = b
    return (la == lb and oa['ticks'] == ob['ticks'] and
            np.array_equal(oa['partials'].view(np.uint64), ob['partials'].view(np.uint64)) and
            np.array_equal(oa['safety_partials'].view(np.uint64), ob['safety_partials'].view(np.uint64)) and
            all(_tsame(t, eb.state[n]) for n, t in ea.state.items()))


@pytest.mark.parametrize('scenario', ['stage1', 'stage2'])
def test_non_binding_limits_change_nothing(built, scenario):
    """10 m/s^2 and 20 rad/s^2 reach any command in one tick: the same env launches, partials and final state as no
    limits at all"""
    a = _evaluate(None, scenario=scenario)
    b = _evaluate(LOOSE, scenario=scenario)
    assert _same_run(a, b)
    assert 'dynamics' not in a[1] and b[1]['dynamics'] == dict(LOOSE, linear=[10.0, 10.0], angular=[20.0, 20.0],
                                                               stream_id=0)


NOISE = dict(range_sigma=0.05, dropout=0.1, v_gain_sigma=0.1, w_gain_sigma=0.1, seed=9)
LATENCY = dict(scan_delay=(0, 2), command_delay=(1, 2), seed=4)


@pytest.mark.parametrize('extra', ['alone', 'noise_latency', 'nh_orca'])
def test_binding_limits_deterministic_and_effective(built, extra):
    kw = dict(noise_kw=NOISE, latency_kw=LATENCY) if extra == 'noise_latency' else \
        dict(scenario='stage2', worlds=2, baseline=True) if extra == 'nh_orca' else {}
    a = _evaluate(RANGED, **kw)
    b = _evaluate(RANGED, **kw)
    assert _same_run(a, b)
    assert a[1]['dynamics']['linear'] == [0.5, 2.0]
    assert not _tsame(a[0].state['pose'], _evaluate(dict(RANGED, seed=5), **kw)[0].state['pose'])
    assert not _tsame(a[0].state['pose'], _evaluate(None, **kw)[0].state['pose'])
    if extra == 'noise_latency':
        assert 'noise' in a[1] and 'latency' in a[1]


def test_dynamics_of_another_env_refused(built):
    from rl_collision_avoidance_b200.dynamics import Dynamics, DynamicsParams
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=1, seed=1, auto_reset=1)
    other = StageWorld(512, scenario='stage1', num_worlds=1, seed=1, auto_reset=1)
    with pytest.raises(ValueError, match='another env'):
        evaluate(env, _policy('stage1_2.pth', env.N), 1, 5, dynamics=Dynamics(other, DynamicsParams(**BOTH)))


def _rollout(envs, H, params, horizons=2):
    """trainer.run's rollout loop with the policy's sampled actions, under limits; the FIFO checked per horizon"""
    from rl_collision_avoidance_b200.model.ppo import generate_action
    from rl_collision_avoidance_b200.trainer import Rollout, compose
    N = sum(e.N for e in envs)
    pol = _policy('stage2.pth', N)
    ro = Rollout(H, N, 512, 'cuda')
    comps = compose(envs, ro, dynamics=params)
    for c in comps:
        c.start()
    resets = 0
    for _ in range(horizons):
        for t in range(H):
            generate_action(env=envs[0], state_list=(ro.stacks[t], ro.gs[t]), policy=pol,
                            action_bound=[[0, -1], [1, 1]],
                            out={'value': ro.values[t], 'action': ro.actions[t], 'logprob': ro.logprobs[t],
                                 'scaled': ro.scaled})
            for c in comps:
                c.tick(t)
        torch.cuda.synchronize()
        resets += _check_fifo(ro, H)
        ro.stacks[0].copy_(ro.stacks[H])
        ro.gs[0].copy_(ro.gs[H])
    return comps, ro, resets


def test_rollout_fifo_under_limits_stage1(built):
    from rl_collision_avoidance_b200.dynamics import DynamicsParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=2, auto_reset=1)
    comps, ro, resets = _rollout([env], 64, DynamicsParams(**RANGED))
    assert 0 < resets < 128 * env.N // 10
    lim = comps[0].dynamics.limits
    assert bool((lim[:, 0] >= 0.5).all() and (lim[:, 0] <= 2.0).all() and (lim[:, 1] >= 1.0).all())
    assert comps[0].dynamics.calls == 128


def test_rollout_fifo_under_limits_random_and_mix(built):
    from rl_collision_avoidance_b200.dynamics import DynamicsParams
    from test_mix_gpu import _envs
    comps, ro, resets = _rollout(_envs(seed=1, names=('random',)), 40, DynamicsParams(**RANGED))
    assert resets > 0
    comps, ro, resets = _rollout(_envs(seed=1), 40, DynamicsParams(**RANGED))
    assert resets > 0
    assert [c.dynamics.stream_id for c in comps] == [0, 1, 2]
    assert all(c.dynamics.calls == 80 for c in comps)


def _train(envs, stage, updates, params, seed=0):
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.trainer import run
    N = sum(e.N for e in envs)
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(256, N))
    policy.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth' if stage == 2 else 'stage1_2.pth'),
                                      map_location='cuda'))
    before = policy.flat.clone()
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=32, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=256, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=envs[0].num_env, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    gen = torch.Generator(device='cuda').manual_seed(seed)
    stats = run(env=envs if len(envs) > 1 else envs[0], policy=policy, policy_path=None, action_bound=[[0, -1], [1, 1]],
                optimizer=opt, hp=hp, stage=stage, max_updates=updates, generator=gen, dynamics=params)
    assert len(stats) == updates and all(np.isfinite(s['losses']).all() for s in stats)
    assert float((policy.flat - before).abs().max()) > 0 and torch.isfinite(policy.flat).all()
    return policy


def test_ppo_updates_under_limits(built):
    from rl_collision_avoidance_b200.dynamics import DynamicsParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from test_mix_gpu import _envs
    p = DynamicsParams(**RANGED)
    a = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    b = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    assert _tsame(a.flat, b.flat)                     # deterministic under limits
    c = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, None)
    assert not _tsame(a.flat, c.flat)                 # and the limits change what is learnt
    _train(_envs(seed=2, names=('random',)), 2, 2, p)
    _train(_envs(seed=2), 2, 2, p)
