"""Sensor and actuation noise on the device (DESIGN.md §9p): the kernels against the host twins bit for bit at the
bench shape, at R = 1, 44 and 64 and at unaligned beam counts and stacks; evaluate() under noise (deterministic, the
true scan / goal / state untouched, zero settings launching nothing); PPO updates under noise on stage 1, on random
layouts with re-layouts and on a mix, with the FIFO invariants of the rollout's stacks."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
FULL = dict(range_sigma=0.1, dropout=0.1, v_gain_sigma=0.2, w_gain_sigma=0.1, seed=2 ** 40 + 17)


def _bits(t):
    a = t.cpu().numpy() if isinstance(t, torch.Tensor) else t
    return np.ascontiguousarray(a).view(np.uint32)


def _cfg(R, W, B, world_offset=0):
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario
    cfg = fill_config(_lib.EnvConfig(), make_scenario('stage1'), num_worlds=W, beams=B, world_offset=world_offset)
    cfg.robots_per_world = R
    return cfg


def _scan_device(cfg, p, draw, stack, flags, stream_id):
    import ctypes as C
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    fp = C.c_void_p(flags.data_ptr()) if flags is not None else None
    _lib.check(lib.rlca_noise_scan(C.byref(cfg), C.byref(p.struct(stream_id)), draw, fp,
                                   C.c_void_p(stack.data_ptr()), None))


def _action_device(cfg, p, draw, cmd, out, stream_id):
    import ctypes as C
    from rl_collision_avoidance_b200 import _lib
    _lib.check(_lib.load().rlca_noise_action(C.byref(cfg), C.byref(p.struct(stream_id)), draw,
                                             C.c_void_p(cmd.data_ptr()), C.c_void_p(out.data_ptr()), None))


@pytest.mark.parametrize('R,W,B,offset', [(24, 171, 512, 0), (1, 300, 512, 5), (44, 12, 512, 3), (64, 9, 512, 0),
                                          (24, 10, 500, 0), (7, 5, 13, 2), (24, 10, 512, 1)])
def test_kernels_equal_host_twins(built, R, W, B, offset):
    """offset: the stack starts `offset` floats into its allocation (1 and 2 leave it unaligned: the scalar path)"""
    from rl_collision_avoidance_b200.noise import NoiseParams, action_host, scan_host
    cfg = _cfg(R, W, B, world_offset=offset * 10)
    N = R * W
    rng = np.random.default_rng(R * 1000 + B)
    host = (rng.uniform(0.05, 5.95, (N, 3, B)) / 6.0 - 0.5).astype(np.float32)
    host[rng.random((N, 3, B)) < 0.2] = np.float32(0.5)
    flags = np.zeros((N, 4), np.uint8)
    flags[rng.random(N) < 0.25, 3] = 1
    cmd = np.stack([rng.uniform(-0.2, 1.2, N), rng.uniform(-1.2, 1.2, N)], 1).astype(np.float32)
    cmd[::7] = 0.0
    for k, p in enumerate((NoiseParams(**FULL), NoiseParams(range_sigma=0.3, seed=1),
                           NoiseParams(dropout=0.5, seed=2), NoiseParams(seed=3))):
        for fl in (flags, None):
            buf = torch.zeros(N * 3 * B + offset, device='cuda')
            dev = buf[offset:].view(N, 3, B)
            dev.copy_(torch.from_numpy(host))
            h = host.copy()
            scan_host(cfg, p, 1000 + k, h, fl, stream_id=k)
            _scan_device(cfg, p, 1000 + k, dev, None if fl is None else torch.from_numpy(fl).cuda(), k)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(dev), _bits(h)), (k, fl is None)
        out = torch.empty(N, 2, device='cuda')
        cin = torch.from_numpy(cmd).cuda()
        _action_device(cfg, p, 7 + k, cin, out, k)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(out), _bits(action_host(cfg, p, 7 + k, cmd, stream_id=k))), k
        assert np.array_equal(_bits(cin), _bits(cmd))


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cuda'))
    return pol


def _evaluate(noise_kw, scenario='stage1', worlds=6, ticks=80, seed=3):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate
    from rl_collision_avoidance_b200.noise import Noise, NoiseParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])
    noise = None if noise_kw is None else Noise(env, NoiseParams(**noise_kw))
    before = env.launch_count
    out = evaluate(env, _policy('stage1_2.pth', env.N), 2, ticks, check_every=20, safety=0.1, noise=noise)
    torch.cuda.synchronize()
    return env, out, env.launch_count - before


def test_evaluate_under_noise_is_deterministic(built):
    """Two runs with one noise seed: the same partials, safety partials and final poses bit for bit; another seed
    drives the robots elsewhere"""
    ea, a, _ = _evaluate(FULL)
    eb, b, _ = _evaluate(FULL)
    assert a['ticks'] == b['ticks']
    assert np.array_equal(a['partials'].view(np.uint64), b['partials'].view(np.uint64))
    assert np.array_equal(a['safety_partials'].view(np.uint64), b['safety_partials'].view(np.uint64))
    assert _tsame(ea.state['pose'], eb.state['pose'])
    assert a['noise'] == dict(FULL, stream_id=0)
    ec, _, _ = _evaluate(dict(FULL, seed=5))
    assert not _tsame(ea.state['pose'], ec.state['pose'])


def test_zero_noise_changes_nothing(built):
    """All-zero settings issue no noise launch: the same env launches and the same partials as no noise at all"""
    _, a, la = _evaluate(None)
    _, b, lb = _evaluate({})
    assert la == lb and a['ticks'] == b['ticks']
    assert np.array_equal(a['partials'].view(np.uint64), b['partials'].view(np.uint64))
    assert np.array_equal(a['safety_partials'].view(np.uint64), b['safety_partials'].view(np.uint64))
    assert 'noise' not in a and b['noise']['range_sigma'] == 0.0


def test_noise_never_touches_the_true_scan_goal_or_state(built):
    """Per tick of a stage-1 run: the noise calls leave env.obs, env.gs, the state and the command bit for bit, the
    tick writes the true scan into the stack and the noise then perturbs it there only."""
    from rl_collision_avoidance_b200.model.ppo import generate_action_no_sampling
    from rl_collision_avoidance_b200.noise import Noise, NoiseParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)
    noise = Noise(env, NoiseParams(**FULL))
    pol = _policy('stage1_2.pth', env.N)
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, 512, device='cuda')]
    noise.scan(stacks[0])
    for tick in range(40):
        k = tick & 1
        _, scaled = generate_action_no_sampling(env=env, state_list=(stacks[k], env.get_local_goal(),
                                                                     env.get_self_speed()),
                                                policy=pol, action_bound=[[0, -1], [1, 1]])
        keep = scaled.clone()
        executed = noise.action(scaled)
        assert _tsame(scaled, keep) and executed.data_ptr() != scaled.data_ptr()
        env.control_vel(executed, stack_in=stacks[k], stack_out=stacks[1 - k])
        snap = {n: t.clone() for n, t in (('obs', env.obs), ('gs', env.gs), ('flags', env.flags))}
        snap.update({'state_' + n: t.clone() for n, t in env.state.items()})
        written = stacks[1 - k][:, 2].clone()
        noise.scan(stacks[1 - k], env.flags)
        torch.cuda.synchronize()
        for n, t in (('obs', env.obs), ('gs', env.gs), ('flags', env.flags)):
            assert _tsame(t, snap[n]), (tick, n)
        for n, t in env.state.items():
            assert _tsame(t, snap['state_' + n]), (tick, n)
        assert _tsame(written, env.obs)
        assert not _tsame(stacks[1 - k][:, 2], env.obs)
    assert noise.scan_draws == 41 and noise.action_draws == 40


def _tsame(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _check_fifo(ro, H, name=''):
    """frames 0-1 of slot t + 1 are frames 1-2 of slot t for rows that were not reset; reset rows hold three copies"""
    for t in range(H):
        fresh = ro.flags[t, :, 3] != 0
        nxt, cur = ro.stacks[t + 1], ro.stacks[t]
        assert _tsame(nxt[~fresh, 0:2], cur[~fresh, 1:3]), (name, t)
        assert _tsame(nxt[fresh, 0], nxt[fresh, 2]) and _tsame(nxt[fresh, 1], nxt[fresh, 2]), (name, t)
    return int((ro.flags[:, :, 3] != 0).sum())


def _rollout(envs, H, params, horizons=2, seed=0):
    """trainer.run's rollout loop with the policy's sampled actions, under noise; returns the rollout after each
    horizon's FIFO check and the number of reset rows seen"""
    from rl_collision_avoidance_b200.model.ppo import generate_action
    from rl_collision_avoidance_b200.trainer import Rollout, compose
    N = sum(e.N for e in envs)
    pol = _policy('stage2.pth', N)
    ro = Rollout(H, N, 512, 'cuda')
    comps = compose(envs, ro, params)
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


def test_rollout_fifo_under_noise_stage1(built):
    from rl_collision_avoidance_b200.noise import NoiseParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=2, auto_reset=1)
    comps, ro, resets = _rollout([env], 64, NoiseParams(**FULL))
    assert resets > 0
    # the stacks really are noisy: the newest frame differs from the true scan the env holds
    assert not _tsame(ro.stacks[64][:, 2], env.obs)


def test_rollout_fifo_under_noise_random_and_mix(built):
    from rl_collision_avoidance_b200.noise import NoiseParams
    from test_mix_gpu import _envs
    comps, ro, resets = _rollout(_envs(seed=1, names=('random',)), 40, NoiseParams(**FULL), horizons=2)
    assert resets > 0
    envs = _envs(seed=1)
    comps, ro, resets = _rollout(envs, 40, NoiseParams(**FULL), horizons=2)
    assert resets > 0
    assert [c.noise.stream_id for c in comps] == [0, 1, 2]
    assert all(c.noise.scan_draws == 81 and c.noise.action_draws == 80 for c in comps)


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
                optimizer=opt, hp=hp, stage=stage, max_updates=updates, generator=gen, noise=params)
    assert len(stats) == updates and all(np.isfinite(s['losses']).all() for s in stats)
    assert float((policy.flat - before).abs().max()) > 0 and torch.isfinite(policy.flat).all()
    return policy


def test_ppo_updates_under_noise(built):
    from rl_collision_avoidance_b200.noise import NoiseParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from test_mix_gpu import _envs
    p = NoiseParams(**FULL)
    a = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    b = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    assert _tsame(a.flat, b.flat)                     # deterministic under noise
    c = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, None)
    assert not _tsame(a.flat, c.flat)                 # and the noise changes what is learnt
    _train(_envs(seed=2, names=('random',)), 2, 2, p)
    _train(_envs(seed=2), 2, 2, p)
