"""Sensing and command latency on the device (DESIGN.md §9q): the kernels against the host twins bit for bit over
20-tick sequences with resets at the bench shape, at R = 1, 44 and 64, at 500 and 13 beams and on unaligned stacks;
stage 1 end to end, tick by tick (the delivered frame and the driven speed against the true history, the env's own
buffers untouched); evaluate() under latency, alone and with noise; rollouts with the FIFO invariants and PPO updates
under latency on stage 1, on random layouts with re-layouts and on a mix."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
RANGED = dict(scan_delay=(0, 4), command_delay=(1, 3), seed=2 ** 40 + 17)


def _bits(t):
    a = t.cpu().numpy() if isinstance(t, torch.Tensor) else t
    return np.ascontiguousarray(a).view(np.uint32)


def _tsame(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _cfg(R, W, B, world_offset=0):
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario
    cfg = fill_config(_lib.EnvConfig(), make_scenario('stage1'), num_worlds=W, beams=B, world_offset=world_offset)
    cfg.robots_per_world = R
    return cfg


def _device_state(N, B, p):
    from rl_collision_avoidance_b200 import _lib
    bufs = (torch.zeros(N, p.scan_delay[1] + 1, B, device='cuda'), torch.zeros(N, p.command_delay[1] + 1, 2,
                                                                               device='cuda'),
            torch.zeros(N, dtype=torch.uint8, device='cuda'), torch.zeros(N, dtype=torch.uint8, device='cuda'))
    return bufs, _lib.LatencyState(*(b.data_ptr() for b in bufs))


def _scan_device(cfg, p, st, draw, stack, flags, stream_id):
    import ctypes as C
    from rl_collision_avoidance_b200 import _lib
    fp = C.c_void_p(flags.data_ptr()) if flags is not None else None
    _lib.check(_lib.load().rlca_latency_scan(C.byref(cfg), C.byref(p.struct(stream_id)), C.byref(st), draw, fp,
                                             C.c_void_p(stack.data_ptr()), None))


def _action_device(cfg, p, st, draw, flags, cmd, out, stream_id):
    import ctypes as C
    from rl_collision_avoidance_b200 import _lib
    fp = C.c_void_p(flags.data_ptr()) if flags is not None else None
    _lib.check(_lib.load().rlca_latency_action(C.byref(cfg), C.byref(p.struct(stream_id)), C.byref(st), draw, fp,
                                               C.c_void_p(cmd.data_ptr()), C.c_void_p(out.data_ptr()), None))


@pytest.mark.parametrize('R,W,B,offset', [(24, 171, 512, 0), (1, 300, 512, 5), (44, 12, 512, 3), (64, 9, 512, 0),
                                          (24, 10, 500, 0), (7, 5, 13, 2), (24, 10, 512, 1), (24, 10, 512, 2),
                                          (24, 10, 512, 3)])
def test_kernels_equal_host_twins(built, R, W, B, offset):
    """20 ticks: the first calls without flags, then random resets (or, for half the settings, no flags at all on
    later calls: every row fresh).  offset: the stack starts `offset` floats into its allocation (1-3: the scalar
    path)."""
    from rl_collision_avoidance_b200.latency import HostState, LatencyParams, action_host, scan_host
    cfg = _cfg(R, W, B, world_offset=offset * 10)
    N = R * W
    rng = np.random.default_rng(R * 1000 + B + offset)
    for k, (p, with_flags) in enumerate(((LatencyParams(**RANGED), True), (LatencyParams(scan_delay=(8, 8),
                                                                                         command_delay=(0, 8), seed=1),
                                                                           True),
                                         (LatencyParams(scan_delay=(2, 2), seed=2), False),
                                         (LatencyParams(command_delay=(3, 3), seed=3), False))):
        hs = HostState(cfg, p)
        bufs, st = _device_state(N, B, p)
        buf = torch.zeros(N * 3 * B + offset, device='cuda')
        dev = buf[offset:].view(N, 3, B)
        host = np.repeat(((rng.uniform(0.05, 5.95, (N, B)) / 6.0) - 0.5).astype(np.float32)[:, None], 3, 1)
        dev.copy_(torch.from_numpy(host))
        scan_host(cfg, p, hs, 0, host, None, stream_id=k)
        _scan_device(cfg, p, st, 0, dev, None, k)
        out = torch.empty(N, 2, device='cuda')
        prev = None
        for t in range(20):
            cmd = np.stack([rng.uniform(-0.2, 1.2, N), rng.uniform(-1.2, 1.2, N)], 1).astype(np.float32)
            cin = torch.from_numpy(cmd).cuda()
            ex = action_host(cfg, p, hs, t, cmd, prev, stream_id=k)
            _action_device(cfg, p, st, t, None if prev is None else torch.from_numpy(prev).cuda(), cin, out, k)
            flags = np.zeros((N, 4), np.uint8)
            flags[rng.random(N) < 0.15, 3] = 1
            newest = ((rng.uniform(0.05, 5.95, (N, B)) / 6.0) - 0.5).astype(np.float32)
            host = np.concatenate([host[:, 1:3], newest[:, None]], 1)
            host[flags[:, 3] != 0, 0:2] = newest[flags[:, 3] != 0, None]
            dev.copy_(torch.from_numpy(host))
            fl = flags if with_flags else None
            scan_host(cfg, p, hs, t + 1, host, fl, stream_id=k)
            _scan_device(cfg, p, st, t + 1, dev, None if fl is None else torch.from_numpy(fl).cuda(), k)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(out), _bits(ex)), (k, t)
            assert np.array_equal(_bits(cin), _bits(cmd))
            assert np.array_equal(_bits(dev), _bits(host)), (k, t)
            prev = fl
        if p.scan_on:
            assert np.array_equal(bufs[2].cpu().numpy(), hs.scan_delay)
            assert np.array_equal(_bits(bufs[0]), _bits(hs.scan_ring))
        if p.command_on:
            assert np.array_equal(bufs[3].cpu().numpy(), hs.cmd_delay)
            assert np.array_equal(_bits(bufs[1]), _bits(hs.cmd_ring))


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cuda'))
    return pol


@pytest.mark.parametrize('kw', [dict(scan_delay=(3, 3), command_delay=(2, 2), seed=4), RANGED])
def test_stage1_end_to_end_against_the_true_history(built, kw):
    """Stage 1 re-spawns inside the tick.  Per tick: the newest frame the policy reads is env.obs of d ticks earlier,
    or the episode's first scan; the speed in gs is the command issued l ticks earlier, or the episode's first command,
    clipped; the latency calls leave env.obs, env.gs, the flags and the state bit for bit."""
    from rl_collision_avoidance_b200.latency import Latency, LatencyParams
    from rl_collision_avoidance_b200.model.ppo import generate_action_no_sampling
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)
    lat = Latency(env, LatencyParams(**kw))
    pol = _policy('stage1_2.pth', env.N)
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    obs = [env.get_laser_observation().clone()]        # obs[k]: the true scan after k ticks
    stacks = [obs[0][:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, 512, device='cuda')]
    lat.scan(stacks[0])
    d, l = lat.scan_delays.long(), lat.command_delays.long()
    assert int(d.min()) >= kw['scan_delay'][0] and int(d.max()) <= kw['scan_delay'][1]
    scan_start = torch.zeros(env.N, dtype=torch.long, device='cuda')
    cmd_start = torch.zeros(env.N, dtype=torch.long, device='cuda')
    issued = []
    lo = torch.tensor([env.cfg.v_min, env.cfg.w_min], device='cuda')
    hi = torch.tensor([env.cfg.v_max, env.cfg.w_max], device='cuda')
    resets = 0
    rows = torch.arange(env.N, device='cuda')
    for tick in range(60):
        k = tick & 1
        _, scaled = generate_action_no_sampling(env=env, state_list=(stacks[k], env.get_local_goal(),
                                                                     env.get_self_speed()),
                                                policy=pol, action_bound=[[0, -1], [1, 1]])
        scaled = scaled + 0.3 * torch.randn_like(scaled)   # commands far from the bound and out of it
        issued.append(scaled.clone())
        prev = env.flags.clone() if tick > 0 else None
        if prev is not None:
            cmd_start = torch.where(prev[:, 3] != 0, tick, cmd_start)
        snap = {'obs': env.obs.clone(), 'gs': env.gs.clone(), 'flags': env.flags.clone()}
        snap.update({'state_' + n: t.clone() for n, t in env.state.items()})
        executed = lat.action(scaled, prev)
        l = lat.command_delays.long()
        assert _tsame(scaled, issued[-1])
        for n in ('obs', 'gs', 'flags'):
            assert _tsame(getattr(env, n), snap[n]), (tick, n)
        env.control_vel(executed, stack_in=stacks[k], stack_out=stacks[1 - k])
        obs.append(env.obs.clone())
        snap = {'obs': env.obs.clone(), 'gs': env.gs.clone(), 'flags': env.flags.clone()}
        snap.update({'state_' + n: t.clone() for n, t in env.state.items()})
        lat.scan(stacks[1 - k], env.flags)
        torch.cuda.synchronize()
        for n in ('obs', 'gs', 'flags'):
            assert _tsame(getattr(env, n), snap[n]), (tick, n)
        for n, t in env.state.items():
            assert _tsame(t, snap['state_' + n]), (tick, n)
        fresh = env.flags[:, 3] != 0
        resets += int(fresh.sum())
        scan_start = torch.where(fresh, tick + 1, scan_start)
        d = lat.scan_delays.long()
        src = torch.maximum(tick + 1 - d, scan_start)
        want = torch.stack(obs)[src, rows]
        assert _tsame(stacks[1 - k][:, 2], want), tick
        # the speed the tick drove with: the clipped command of l ticks earlier, or the episode's first (rows the tick
        # did not re-spawn)
        past = torch.stack(issued)[torch.maximum(tick - l, cmd_start), rows]
        want_cmd = torch.maximum(torch.minimum(past, hi), lo)
        keep = ~fresh
        assert torch.equal(env.gs[keep, 2:4], want_cmd[keep]), tick
    assert 0 < resets < 60 * env.N // 10          # re-spawns stay rare: no robot is held in a crash
    assert lat.scan_calls == 61 and lat.action_calls == 60
    if kw['scan_delay'][1] > kw['scan_delay'][0]:
        assert len(set(lat.scan_delays.tolist())) > 1


def _evaluate(latency_kw, noise_kw=None, scenario='stage1', worlds=6, ticks=80, seed=3):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate
    from rl_collision_avoidance_b200.latency import Latency, LatencyParams
    from rl_collision_avoidance_b200.noise import Noise, NoiseParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])
    lat = None if latency_kw is None else Latency(env, LatencyParams(**latency_kw))
    noise = None if noise_kw is None else Noise(env, NoiseParams(**noise_kw))
    before = env.launch_count
    out = evaluate(env, _policy('stage1_2.pth', env.N), 2, ticks, check_every=20, safety=0.1, noise=noise,
                   latency=lat)
    torch.cuda.synchronize()
    return env, out, env.launch_count - before


NOISE = dict(range_sigma=0.05, dropout=0.1, v_gain_sigma=0.1, w_gain_sigma=0.1, seed=9)


@pytest.mark.parametrize('noise_kw', [None, NOISE])
def test_evaluate_under_latency_is_deterministic(built, noise_kw):
    ea, a, _ = _evaluate(RANGED, noise_kw)
    eb, b, _ = _evaluate(RANGED, noise_kw)
    assert a['ticks'] == b['ticks']
    assert np.array_equal(a['partials'].view(np.uint64), b['partials'].view(np.uint64))
    assert np.array_equal(a['safety_partials'].view(np.uint64), b['safety_partials'].view(np.uint64))
    assert _tsame(ea.state['pose'], eb.state['pose'])
    assert a['latency'] == {'scan_delay': [0, 4], 'command_delay': [1, 3], 'seed': RANGED['seed'], 'stream_id': 0}
    ec, c, _ = _evaluate(dict(RANGED, seed=5), noise_kw)
    assert not _tsame(ea.state['pose'], ec.state['pose'])
    en, n, _ = _evaluate(None, noise_kw)
    assert not _tsame(ea.state['pose'], en.state['pose'])


@pytest.mark.parametrize('noise_kw', [None, NOISE])
def test_zero_delays_change_nothing(built, noise_kw):
    """delays of 0 issue no latency launch: the same env launches and the same partials as no latency at all"""
    _, a, la = _evaluate(None, noise_kw)
    _, b, lb = _evaluate(dict(seed=3), noise_kw)
    assert la == lb and a['ticks'] == b['ticks']
    assert np.array_equal(a['partials'].view(np.uint64), b['partials'].view(np.uint64))
    assert np.array_equal(a['safety_partials'].view(np.uint64), b['safety_partials'].view(np.uint64))
    assert 'latency' not in a and b['latency']['scan_delay'] == [0, 0]


def test_command_latency_with_a_baseline(built):
    """command latency applies to the ORCA baselines; scan delay is refused"""
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.latency import Latency, LatencyParams
    from rl_collision_avoidance_b200.orca import OrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage2', num_worlds=2, seed=1, auto_reset=2)
    ctl = OrcaController(env)
    with pytest.raises(ValueError, match='do not read the scan'):
        evaluate(env, ctl, 1, 10, latency=Latency(env, LatencyParams(scan_delay=(1, 1))))
    a = evaluate(env, ctl, 1, 60, check_every=20, latency=Latency(env, LatencyParams(command_delay=(2, 2))))
    pa = env.state['pose'].clone()
    b = evaluate(env, ctl, 1, 60, check_every=20)
    assert a['latency']['command_delay'] == [2, 2] and 'latency' not in b
    assert not _tsame(pa, env.state['pose'])


def _check_fifo(ro, H):
    """frames 0-1 of slot t + 1 are frames 1-2 of slot t for rows that were not reset; reset rows hold three copies"""
    for t in range(H):
        fresh = ro.flags[t, :, 3] != 0
        nxt, cur = ro.stacks[t + 1], ro.stacks[t]
        assert _tsame(nxt[~fresh, 0:2], cur[~fresh, 1:3]), t
        assert _tsame(nxt[fresh, 0], nxt[fresh, 2]) and _tsame(nxt[fresh, 1], nxt[fresh, 2]), t
    return int((ro.flags[:, :, 3] != 0).sum())


def _rollout(envs, H, params, horizons=2):
    """trainer.run's rollout loop with the policy's sampled actions, under latency; the FIFO checked per horizon"""
    from rl_collision_avoidance_b200.model.ppo import generate_action
    from rl_collision_avoidance_b200.trainer import Rollout, compose
    N = sum(e.N for e in envs)
    pol = _policy('stage2.pth', N)
    ro = Rollout(H, N, 512, 'cuda')
    comps = compose(envs, ro, latency=params)
    for c in comps:
        c.start()
    assert _tsame(ro.stacks[0][:, 0], ro.stacks[0][:, 2]) and _tsame(ro.stacks[0][:, 1], ro.stacks[0][:, 2])
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


def test_rollout_fifo_under_latency_stage1(built):
    from rl_collision_avoidance_b200.latency import LatencyParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=2, auto_reset=1)
    comps, ro, resets = _rollout([env], 64, LatencyParams(**RANGED))
    assert 0 < resets < 128 * env.N // 10
    d = comps[0].latency.scan_delays
    stale = (ro.stacks[64][:, 2] != env.obs).any(1)
    assert int(stale[d > 0].sum()) > int((d > 0).sum()) // 2      # most delayed rows do not read the true scan
    assert not stale[d == 0].any()


def test_rollout_fifo_under_latency_random_and_mix(built):
    from rl_collision_avoidance_b200.latency import LatencyParams
    from test_mix_gpu import _envs
    comps, ro, resets = _rollout(_envs(seed=1, names=('random',)), 40, LatencyParams(**RANGED))
    assert resets > 0
    comps, ro, resets = _rollout(_envs(seed=1), 40, LatencyParams(**RANGED))
    assert resets > 0
    assert [c.latency.stream_id for c in comps] == [0, 1, 2]
    assert all(c.latency.scan_calls == 81 and c.latency.action_calls == 80 for c in comps)


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
                optimizer=opt, hp=hp, stage=stage, max_updates=updates, generator=gen, latency=params)
    assert len(stats) == updates and all(np.isfinite(s['losses']).all() for s in stats)
    assert float((policy.flat - before).abs().max()) > 0 and torch.isfinite(policy.flat).all()
    return policy


def test_ppo_updates_under_latency(built):
    from rl_collision_avoidance_b200.latency import LatencyParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from test_mix_gpu import _envs
    p = LatencyParams(**RANGED)
    a = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    b = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    assert _tsame(a.flat, b.flat)                     # deterministic under latency
    c = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, None)
    assert not _tsame(a.flat, c.flat)                 # and the latency changes what is learnt
    _train(_envs(seed=2, names=('random',)), 2, 2, p)
    _train(_envs(seed=2), 2, 2, p)
