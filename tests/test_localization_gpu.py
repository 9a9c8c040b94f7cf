"""Localization error on the device (DESIGN.md §9s): the kernel against the host twin bit for bit over 20-tick sequences
with resets at the bench shape and at R = 1, 44 and 64, in place and out of place, and on gs slices of a mix's rollout;
stage 1 tick by tick (the env's gs, obs and state equal a run without the error, re-spawned rows get a fresh error on
the tick they re-spawn, zero pose error gives the tick's local goal); evaluate() alone, with noise, latency and
dynamics, and with non-cooperative robots, its trackers equal to a run fed the same actions without the error; rollouts
whose gs is what the twin computes from the truth, and PPO updates on stage 1, on random layouts and on a mix."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from test_latency_gpu import _bits, _cfg, _check_fifo, _policy, _tsame

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
RANGED = dict(pose_sigma=(0.1, 0.3), heading_sigma=(0.05, 0.15), correlation_time=2.0, speed_sigma=(0.05, 0.1),
              seed=2 ** 40 + 17)
OFFSET = dict(pose_sigma=(0.3, 0.3), heading_sigma=(0.1, 0.1), correlation_time=math.inf, seed=5)
SPEED = dict(speed_sigma=(0.1, 0.2), correlation_time=0.0, seed=6)


def _observe_device(cfg, p, bufs, draw, flags, pose, goal, gs_in, gs_out, stream_id):
    from rl_collision_avoidance_b200 import _lib
    st = _lib.LocalizationState(*(b.data_ptr() for b in bufs))
    env = _lib.EnvState(pose.data_ptr(), goal.data_ptr(), None, None)
    fp = C.c_void_p(flags.data_ptr()) if flags is not None else None
    _lib.check(_lib.load().rlca_localization_observe(C.byref(cfg), C.byref(p.struct(stream_id)), C.byref(st), draw,
                                                     fp, C.byref(env), C.c_void_p(gs_in.data_ptr()),
                                                     C.c_void_p(gs_out.data_ptr()), None))


@pytest.mark.parametrize('R,W,offset', [(24, 171, 0), (1, 300, 5), (44, 12, 3), (64, 9, 0), (24, 10, 2)])
@pytest.mark.parametrize('in_place', [False, True])
def test_kernel_equals_host_twin(built, R, W, offset, in_place):
    """20 ticks: the first call without flags, then random resets; poses near +-pi, goals at the robot's position"""
    from rl_collision_avoidance_b200.localization import HostState, LocalizationParams, observe_host
    from test_localization import _inputs
    cfg = _cfg(R, W, 8, world_offset=offset * 10)
    N = R * W
    rng = np.random.default_rng(R * 1000 + offset)
    for k, kw in enumerate((RANGED, OFFSET, SPEED, dict(RANGED, correlation_time=0.0))):
        p = LocalizationParams(**kw)
        hs = HostState(cfg)
        bufs = (torch.zeros(N, 4, device='cuda'), torch.zeros(N, 2, device='cuda'))
        out = torch.empty(N, 4, device='cuda')
        flags = None
        for t in range(20):
            pose, goal, gs = _inputs(rng, N)
            dp, dg, dgs = (torch.from_numpy(a).cuda() for a in (pose, goal, gs))
            ex = observe_host(cfg, p, hs, t, pose, goal, gs, flags, stream_id=k)
            dst = dgs if in_place else out
            _observe_device(cfg, p, bufs, t, None if flags is None else torch.from_numpy(flags).cuda(), dp, dg, dgs,
                            dst, k)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(dst), _bits(ex)), (k, t)
            if not in_place:
                assert np.array_equal(_bits(dgs), _bits(gs))
            assert np.array_equal(_bits(dp), _bits(pose)) and np.array_equal(_bits(dg), _bits(goal))
            assert np.array_equal(_bits(bufs[0]), _bits(hs.err)), (k, t)
            assert np.array_equal(_bits(bufs[1]), _bits(hs.sigma)), (k, t)
            flags = np.zeros((N, 4), np.uint8)
            flags[rng.random(N) < 0.1, 3] = 1


def test_kernel_on_mix_gs_slices(built):
    """a mix's components own consecutive agent columns of ro.gs: in place on slices at their offsets, each slice
    equals the twin and the columns outside it are untouched"""
    from rl_collision_avoidance_b200.localization import HostState, LocalizationParams, observe_host
    from rl_collision_avoidance_b200.mix import SLICE_ALIGN
    from test_localization import _inputs
    assert SLICE_ALIGN['gs'] == 16
    p = LocalizationParams(**RANGED)
    rng = np.random.default_rng(4)
    parts = [(4, 4), (8, 16), (8, 4), (1, 7)]                 # (R, W) of components side by side
    total = sum(R * W for R, W in parts)
    ro_gs = torch.from_numpy(rng.uniform(-3, 3, (3, total, 4)).astype(np.float32)).cuda()
    a = 0
    for k, (R, W) in enumerate(parts):
        cfg = _cfg(R, W, 8, world_offset=k)
        N = R * W
        pose, goal, gs = _inputs(rng, N)
        view = ro_gs[1, a:a + N]
        view.copy_(torch.from_numpy(gs))
        before = ro_gs.clone()
        bufs = (torch.zeros(N, 4, device='cuda'), torch.zeros(N, 2, device='cuda'))
        _observe_device(cfg, p, bufs, 0, None, torch.from_numpy(pose).cuda(), torch.from_numpy(goal).cuda(), view,
                        view, k)
        ex = observe_host(cfg, p, HostState(cfg), 0, pose, goal, gs, stream_id=k)
        torch.cuda.synchronize()
        assert view.data_ptr() % 16 == 0 and np.array_equal(_bits(view), _bits(ex)), k
        mask = torch.ones(3, total, dtype=torch.bool, device='cuda')
        mask[1, a:a + N] = False
        assert _tsame(ro_gs[mask], before[mask]), k
        a += N


def _snapshot(env):
    snap = {'obs': env.obs.clone(), 'gs': env.gs.clone(), 'flags': env.flags.clone()}
    snap.update({'state_' + n: t.clone() for n, t in env.state.items()})
    return snap


def _same_env(a, b):
    return all(_tsame(a[k], b[k]) for k in a)


@pytest.mark.parametrize('kw', [RANGED, OFFSET, SPEED])
def test_stage1_tick_by_tick(built, kw):
    """Two stage-1 envs driven by the same actions (the policy reading the believed gs, plus noise), one of them with a
    Localization: every tick its env.gs, env.obs, flags and state equal the other's bit for bit; with tau = inf rows
    hold their error until they re-spawn and get a fresh one on that tick; the believed gs equals the twin on host
    copies; with zero pose error the local goal is the tick's"""
    from rl_collision_avoidance_b200.localization import HostState, Localization, LocalizationParams, observe_host
    from rl_collision_avoidance_b200.model.ppo import generate_action_no_sampling
    from rl_collision_avoidance_b200.stage_world import StageWorld
    envs = [StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1) for _ in range(2)]
    p = LocalizationParams(**kw)
    loc = Localization(envs[0], p)
    pol = _policy('stage1_2.pth', envs[0].N)
    gen = torch.Generator(device='cuda').manual_seed(1)
    N = envs[0].N
    stacks = []
    for e in envs:
        e.reset_world()
        e.reset_pose()
        e.generate_goal_point()
        obs = e.get_laser_observation()
        stacks.append([obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(N, 3, 512, device='cuda')])
    hs = HostState(envs[0].cfg)

    def observe(flags):
        e = envs[0]
        host = [t.cpu().numpy() for t in (e.state['pose'], e.state['goal'], e.gs)]
        f = None if flags is None else flags.cpu().numpy()
        before = _snapshot(e)
        gs = loc.observe(flags)
        torch.cuda.synchronize()
        assert _same_env(_snapshot(e), before)
        assert np.array_equal(_bits(gs), _bits(observe_host(e.cfg, p, hs, loc.calls - 1, *host, f)))
        return gs

    gs = observe(None)
    resets = 0
    for tick in range(150):
        k = tick & 1
        _, scaled = generate_action_no_sampling(env=envs[0], state_list=(stacks[0][k], gs[:, 0:2], gs[:, 2:4]),
                                                policy=pol, action_bound=[[0, -1], [1, 1]])
        scaled = (scaled + 0.3 * torch.randn(scaled.shape, device='cuda', generator=gen)).contiguous()
        err_before = loc.errors
        for e, st in zip(envs, stacks):
            e.control_vel(scaled, stack_in=st[k], stack_out=st[1 - k])
        torch.cuda.synchronize()
        assert _same_env(_snapshot(envs[0]), _snapshot(envs[1])), tick
        assert _tsame(stacks[0][1 - k], stacks[1][1 - k]), tick
        gs = observe(envs[0].flags)
        fresh = envs[0].flags[:, 3] != 0
        resets += int(fresh.sum())
        if kw is OFFSET:
            err = loc.errors
            assert _tsame(err[~fresh], err_before[~fresh]), tick
            assert bool((err[fresh] != err_before[fresh]).all()), tick
        if kw is SPEED:
            assert _tsame(gs[:, 0:2], envs[0].gs[:, 0:2]), tick
            assert bool((gs[:, 2:4] != envs[0].gs[:, 2:4]).float().mean() > 0.9), tick
    assert resets > 0


def _evaluate(loc_kw, extra=(), scenario='stage1', worlds=6, ticks=80, seed=3, actions=None, record=None):
    """evaluate() with stage1_2.pth, optionally with noise / latency / dynamics and non-cooperative robots.  `record`
    collects the policy's commands; `actions` replays recorded commands instead of the policy's"""
    import rl_collision_avoidance_b200.evaluation as ev
    from rl_collision_avoidance_b200.dynamics import Dynamics, DynamicsParams
    from rl_collision_avoidance_b200.latency import Latency, LatencyParams
    from rl_collision_avoidance_b200.localization import Localization, LocalizationParams
    from rl_collision_avoidance_b200.noise import Noise, NoiseParams
    from rl_collision_avoidance_b200.orca import NonCooperative
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=seed, auto_reset=ev.AUTO_RESET[scenario])
    kw = {}
    if 'noise' in extra:
        kw['noise'] = Noise(env, NoiseParams(range_sigma=0.05, dropout=0.1, v_gain_sigma=0.1, w_gain_sigma=0.1, seed=9))
    if 'latency' in extra:
        kw['latency'] = Latency(env, LatencyParams(scan_delay=(0, 2), command_delay=(1, 2), seed=4))
    if 'dynamics' in extra:
        kw['dynamics'] = Dynamics(env, DynamicsParams(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=2))
    if 'non_cooperative' in extra:
        kw['non_cooperative'] = NonCooperative(env, ev.non_cooperative_mask(env.cfg.robots_per_world, worlds, 2))
    if loc_kw is not None:
        kw['localization'] = Localization(env, LocalizationParams(**loc_kw))
    pol = _policy('stage1_2.pth', env.N)
    gen = ev.generate_action_no_sampling
    calls = []

    def wrapped(**a):
        calls.append(a['state_list'])
        if actions is not None:
            return None, actions[len(calls) - 1].clone()
        v, scaled = gen(**a)
        if record is not None:
            record.append(scaled.clone())
        return v, scaled

    ev.generate_action_no_sampling = wrapped
    try:
        before = env.launch_count
        out = ev.evaluate(env, pol, 2, ticks, check_every=20, safety=0.1, progress={}, **kw)
    finally:
        ev.generate_action_no_sampling = gen
    torch.cuda.synchronize()
    return env, out, env.launch_count - before, calls


def _same_trackers(a, b):
    ea, oa = a[0], a[1]
    eb, ob = b[0], b[1]
    same = lambda x, y: np.array_equal(np.asarray(x).view(np.uint64), np.asarray(y).view(np.uint64))
    return (oa['ticks'] == ob['ticks'] and same(oa['partials'], ob['partials']) and
            same(oa['safety_partials'], ob['safety_partials']) and
            same(oa['progress_partials'], ob['progress_partials']) and
            all(_tsame(t, eb.state[n]) for n, t in ea.state.items()))


@pytest.mark.parametrize('extra', [(), ('noise', 'latency', 'dynamics'), ('non_cooperative',)])
def test_evaluate_trackers_measure_the_truth(built, extra):
    """evaluate() under localization error: deterministic, the policy reads the believed gs (not env.gs), and the
    episode, safety and progress partials and the final state equal those of a run without the error fed the same
    commands; the same env launches as that run (the localization launch is not the env's)"""
    rec = []
    a = _evaluate(RANGED, extra, record=rec)
    b = _evaluate(RANGED, extra)
    assert _same_trackers(a, b)
    assert a[1]['localization'] == dict(RANGED, pose_sigma=[float(np.float32(0.1)), float(np.float32(0.3))],
                                        heading_sigma=[float(np.float32(0.05)), float(np.float32(0.15))],
                                        speed_sigma=[float(np.float32(0.05)), float(np.float32(0.1))], stream_id=0)
    env = a[0]
    goal = a[3][-1][1]
    assert goal.data_ptr() != env.gs.data_ptr()
    replay = _evaluate(None, extra, actions=rec)
    assert _same_trackers(a, replay) and a[2] == replay[2]
    assert 'localization' not in replay[1]
    plain = _evaluate(None, extra)
    assert not _tsame(a[0].state['pose'], plain[0].state['pose'])


def test_evaluate_refusals(built):
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.localization import Localization, LocalizationParams
    from rl_collision_avoidance_b200.orca import Hybrid, NhOrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage2', num_worlds=1, seed=1, auto_reset=2)
    other = StageWorld(512, scenario='stage2', num_worlds=1, seed=1, auto_reset=2)
    pol = _policy('stage2.pth', env.N)
    with pytest.raises(ValueError, match='another env'):
        evaluate(env, pol, 1, 5, localization=Localization(other, LocalizationParams(**RANGED)))
    loc = Localization(env, LocalizationParams(**RANGED))
    with pytest.raises(ValueError, match='ORCA'):
        evaluate(env, NhOrcaController(env), 1, 5, localization=loc)
    with pytest.raises(ValueError, match='hybrid'):
        evaluate(env, pol, 1, 5, hybrid=Hybrid(env), localization=loc)


def _rollout(envs, H, params, horizons=2):
    """trainer.run's rollout loop under localization error; every observe checked against the twin on host copies of
    the truth it read, so ro.gs holds exactly what the policy reads"""
    from rl_collision_avoidance_b200.localization import HostState, observe_host
    from rl_collision_avoidance_b200.model.ppo import generate_action
    from rl_collision_avoidance_b200.trainer import Rollout, compose
    N = sum(e.N for e in envs)
    pol = _policy('stage2.pth', N)
    ro = Rollout(H, N, 512, 'cuda')
    comps = compose(envs, ro, localization=params)
    checked = [0]
    for c in comps:
        loc, hs = c.localization, HostState(c.env.cfg)
        real = loc.observe

        def observe(flags=None, gs=None, out=None, loc=loc, hs=hs, real=real, e=c.env):
            host = [t.cpu().numpy() for t in (e.state['pose'], e.state['goal'], gs)]
            f = None if flags is None else flags.cpu().numpy()
            res = real(flags, gs=gs, out=out)
            torch.cuda.synchronize()
            assert res is out and out.data_ptr() == gs.data_ptr()
            ex = observe_host(e.cfg, loc.params, hs, loc.calls - 1, *host, f, stream_id=loc.stream_id)
            assert np.array_equal(_bits(res), _bits(ex)), loc.calls
            checked[0] += 1
            return res

        loc.observe = observe
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
    assert checked[0] == len(comps) * (1 + horizons * H)
    return comps, ro, resets


def test_rollout_gs_is_believed_stage1(built):
    from rl_collision_avoidance_b200.localization import LocalizationParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=2, auto_reset=1)
    comps, ro, resets = _rollout([env], 64, LocalizationParams(**RANGED))
    assert resets > 0
    sg = comps[0].localization.sigmas
    assert bool((sg[:, 0] >= np.float32(0.1)).all() and (sg[:, 0] <= np.float32(0.3)).all())


def test_rollout_gs_is_believed_random_and_mix(built):
    from rl_collision_avoidance_b200.localization import LocalizationParams
    from test_mix_gpu import _envs
    comps, ro, resets = _rollout(_envs(seed=1, names=('random',)), 40, LocalizationParams(**RANGED))
    assert resets > 0
    comps, ro, resets = _rollout(_envs(seed=1), 40, LocalizationParams(**RANGED))
    assert resets > 0
    assert [c.localization.stream_id for c in comps] == [0, 1, 2]
    assert all(c.localization.calls == 81 for c in comps)


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
                optimizer=opt, hp=hp, stage=stage, max_updates=updates, generator=gen, localization=params)
    assert len(stats) == updates and all(np.isfinite(s['losses']).all() for s in stats)
    assert float((policy.flat - before).abs().max()) > 0 and torch.isfinite(policy.flat).all()
    return policy


def test_ppo_updates_under_localization_error(built):
    from rl_collision_avoidance_b200.localization import LocalizationParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from test_mix_gpu import _envs
    p = LocalizationParams(**RANGED)
    a = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    b = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, p)
    assert _tsame(a.flat, b.flat)                     # deterministic under the error
    c = _train([StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)], 1, 2, None)
    assert not _tsame(a.flat, c.flat)                 # and the error changes what is learnt
    _train(_envs(seed=2, names=('random',)), 2, 2, p)
    _train(_envs(seed=2), 2, 2, p)
