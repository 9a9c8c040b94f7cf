"""Localization error on the host (DESIGN.md §9s): the host twin of rlca_localization_observe against the numpy
restatement in tests/localization_ref.py, bit for bit, over multi-tick sequences with resets, poses near +-pi and goals
at the robot's position; zero pose error as the tick's own local goal; tau = inf holding the error; draws independent of
the world count and shard and different per stream and seed; the statistics of the error process, the per-episode
sigmas and the speed noise; every invalid argument of the C entries and of the Python layer; the command-line rules of
evaluate.py and the trainers."""
import ctypes as C
import math
import os
import re
import subprocess
import types

import numpy as np
import pytest
from scipy import stats

import localization_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.localization import HostState, Localization, LocalizationParams, observe_host
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(R=4, W=3, world_offset=0):
    cfg = fill_config(_lib.EnvConfig(), make_scenario('stage1'), num_worlds=W, beams=8, world_offset=world_offset)
    cfg.robots_per_world = R
    return cfg


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _inputs(rng, N):
    """env-state pose and goal and the tick's gs: headings up to and across +-pi (and exactly +-pi, -0), goals at the
    robot's position on some rows, speeds with -0"""
    pose = np.zeros((N, 4), np.float32)
    pose[:, 0:2] = rng.uniform(-10, 10, (N, 2))
    pose[:, 2] = rng.uniform(-math.pi, math.pi, N)
    edge = rng.random(N) < 0.2
    pose[edge, 2] = rng.choice(np.array([np.pi, -np.pi, np.nextafter(np.float32(np.pi), 0), -0.0, 0.0], np.float32),
                               int(edge.sum()))
    pose[:, 3] = rng.uniform(0, 5, N)
    goal = np.zeros((N, 4), np.float32)
    goal[:, 0:2] = pose[:, 0:2] + rng.uniform(-6, 6, (N, 2)).astype(np.float32)
    at = rng.random(N) < 0.15
    goal[at, 0:2] = pose[at, 0:2]
    goal[:, 2] = rng.uniform(0, 1, N)
    goal[:, 3] = rng.uniform(-1, 1, N)
    gs = np.zeros((N, 4), np.float32)
    gs[:, 0:2] = rng.uniform(-5, 5, (N, 2))
    gs[:, 2:4] = goal[:, 2:4]
    gs[rng.random(N) < 0.1, 2] = -0.0
    return pose, goal, gs


def _run(R, W, p, ticks, seed=0, world_offset=0, stream=0, reset_p=0.1):
    """ticks of the host twin and of the restatement side by side; asserts bit equality on every call"""
    cfg = _cfg(R, W, world_offset)
    N = R * W
    rng = np.random.default_rng(seed)
    hs = HostState(cfg)
    ref = localization_ref.Localization(R, W, p.pose_sigma, p.heading_sigma, p.correlation_time, p.speed_sigma,
                                        p.seed, cfg.dt, world_offset, stream)
    flags = None
    outs = []
    for t in range(ticks):
        pose, goal, gs = _inputs(rng, N)
        keep = [a.copy() for a in (pose, goal, gs)]
        out = observe_host(cfg, p, hs, t, pose, goal, gs, flags, stream_id=stream)
        assert np.array_equal(_bits(out), _bits(ref.observe(pose, goal, gs, flags))), t
        assert all(np.array_equal(_bits(a), _bits(b)) for a, b in zip((pose, goal, gs), keep))
        assert np.array_equal(_bits(hs.err[:, 0:3]), _bits(ref.err)), t
        assert np.array_equal(_bits(hs.sigma), _bits(ref.sigma)), t
        outs.append(out)
        flags = np.zeros((N, 4), np.uint8)
        flags[rng.random(N) < reset_p, 3] = 1
        flags[rng.random(N) < 0.1, 0] = 1           # done and crashed alone do not start an episode
        flags[rng.random(N) < 0.1, 1] = 1
    return hs, outs


# ------------------------------------------------------------------------------------------------ reference
SETTINGS = [dict(pose_sigma=(0.1, 0.1), heading_sigma=(0.05, 0.05), correlation_time=2.0),
            dict(pose_sigma=(0.05, 0.3), heading_sigma=(0.0, 0.15), correlation_time=0.0),
            dict(pose_sigma=(0.2, 0.2), correlation_time=math.inf, speed_sigma=(0.05, 0.1)),
            dict(heading_sigma=(0.1, 0.3), correlation_time=0.35, speed_sigma=(0.0, 0.2)),
            dict(speed_sigma=(0.1, 0.0)),
            dict(pose_sigma=(0.0, 1.0), heading_sigma=(0.5, 0.5), correlation_time=1e30, speed_sigma=(0.3, 0.3)),
            dict()]


@pytest.mark.parametrize('kw', SETTINGS, ids=lambda d: ','.join('%s=%s' % kv for kv in d.items()) or 'zero')
def test_host_twin_equals_restatement(built, kw):
    p = LocalizationParams(seed=2 ** 40 + 3, **kw)
    hs, _ = _run(5, 3, p, 40, seed=len(kw), world_offset=7, stream=2)
    for (lo, hi), got in ((p.pose_sigma, hs.sigma[:, 0]), (p.heading_sigma, hs.sigma[:, 1])):
        assert got.min() >= lo and got.max() <= hi


def test_host_twin_equals_restatement_many_resets(built):
    p = LocalizationParams(pose_sigma=(0.1, 0.3), heading_sigma=(0.05, 0.15), correlation_time=0.5,
                           speed_sigma=(0.05, 0.1), seed=11)
    _run(8, 4, p, 60, seed=3, reset_p=0.5)
    _run(8, 4, p, 40, seed=4, reset_p=0.0)


# ------------------------------------------------------------------------------------------------ properties
def test_zero_pose_error_gives_the_ticks_local_goal(built):
    """sigma_xy = sigma_theta = 0 with speed noise on: gs.xy is goal_speed of the true pose, bit for bit (-0 included),
    and gs.zw is the true speed plus noise"""
    cfg = _cfg(16, 4)
    N = 64
    rng = np.random.default_rng(5)
    p = LocalizationParams(correlation_time=0.7, speed_sigma=(0.1, 0.2), seed=1)
    hs = HostState(cfg)
    flags = None
    for t in range(10):
        pose, goal, gs = _inputs(rng, N)
        out = observe_host(cfg, p, hs, t, pose, goal, gs, flags)
        s, c = localization_ref.sincos(pose[:, 2])
        assert np.array_equal(_bits(out[:, 0:2]), _bits(localization_ref.goal_speed(pose, goal, s, c))), t
        assert (out[:, 2:4] != gs[:, 2:4]).mean() > 0.95
        assert not hs.err.any()
        flags = np.zeros((N, 4), np.uint8)
        flags[rng.random(N) < 0.2, 3] = 1


def test_zero_settings_are_the_identity_on_the_local_goal(built):
    """with every setting 0 the entry still runs (the Python object launches nothing): gs.xy is the tick's, gs.zw the
    true speed itself"""
    cfg = _cfg(8, 2)
    pose, goal, gs = _inputs(np.random.default_rng(1), 16)
    out = observe_host(cfg, LocalizationParams(), HostState(cfg), 0, pose, goal, gs)
    s, c = localization_ref.sincos(pose[:, 2])
    assert np.array_equal(_bits(out[:, 0:2]), _bits(localization_ref.goal_speed(pose, goal, s, c)))
    assert np.array_equal(_bits(out[:, 2:4]), _bits(gs[:, 2:4]))


def test_constant_offset_held_then_redrawn_on_reset(built):
    """tau = inf: e is bit-identical on every call of an episode and redrawn (with its sigma) when was_reset is set"""
    cfg = _cfg(8, 4)
    N = 32
    p = LocalizationParams(pose_sigma=(0.1, 0.5), heading_sigma=(0.05, 0.2), correlation_time=math.inf, seed=7)
    hs = HostState(cfg)
    rng = np.random.default_rng(2)
    pose, goal, gs = _inputs(rng, N)
    observe_host(cfg, p, hs, 0, pose, goal, gs)
    first, sig = hs.err.copy(), hs.sigma.copy()
    assert (first[:, 0:3] != 0).all()
    none = np.zeros((N, 4), np.uint8)
    none[:, 0:2] = 1                                # done / crashed without a reset change nothing
    for t in range(1, 30):
        observe_host(cfg, p, hs, t, *_inputs(rng, N), none)
        assert np.array_equal(_bits(hs.err), _bits(first)) and np.array_equal(_bits(hs.sigma), _bits(sig)), t
    reset = np.zeros((N, 4), np.uint8)
    reset[::3, 3] = 1
    observe_host(cfg, p, hs, 30, *_inputs(rng, N), reset)
    r = reset[:, 3] != 0
    assert (hs.err[r, 0:3] != first[r, 0:3]).all() and (hs.sigma[r] != sig[r]).all()
    assert np.array_equal(_bits(hs.err[~r]), _bits(first[~r])) and np.array_equal(_bits(hs.sigma[~r]), _bits(sig[~r]))


def test_draws_independent_of_num_worlds_and_shards(built):
    """world k of a 7-world config at offset 0 equals the 1-world config at world_offset k, on every call"""
    R, k = 6, 4
    p = LocalizationParams(pose_sigma=(0.1, 0.3), heading_sigma=(0.05, 0.15), correlation_time=1.0,
                           speed_sigma=(0.05, 0.1), seed=99)
    big, one = _cfg(R, 7), _cfg(R, 1, world_offset=k)
    hb, ho = HostState(big), HostState(one)
    rng = np.random.default_rng(8)
    flags = None
    for t in range(12):
        pose, goal, gs = _inputs(rng, 7 * R)
        sl = slice(k * R, (k + 1) * R)
        ob = observe_host(big, p, hb, t, pose, goal, gs, flags, stream_id=3)
        oo = observe_host(one, p, ho, t, pose[sl], goal[sl], gs[sl], None if flags is None else flags[sl],
                          stream_id=3)
        assert np.array_equal(_bits(ob[sl]), _bits(oo)), t
        assert np.array_equal(_bits(hb.err[sl]), _bits(ho.err)), t
        flags = np.zeros((7 * R, 4), np.uint8)
        flags[rng.random(7 * R) < 0.2, 3] = 1


@pytest.mark.parametrize('change', ['stream', 'seed', 'draw'])
def test_other_stream_seed_or_draw_gives_other_draws(built, change):
    cfg = _cfg(64, 4)
    N = 256
    pose, goal, gs = _inputs(np.random.default_rng(0), N)
    base = dict(pose_sigma=(0.1, 0.3), heading_sigma=(0.05, 0.15), speed_sigma=(0.1, 0.1), seed=5)
    runs = []
    for k in (0, 1):
        p = LocalizationParams(**dict(base, seed=5 + k if change == 'seed' else 5))
        hs = HostState(cfg)
        out = observe_host(cfg, p, hs, k if change == 'draw' else 0, pose, goal, gs,
                           stream_id=k if change == 'stream' else 0)
        runs.append((out, hs.err.copy(), hs.sigma.copy()))
    for a, b in zip(*runs):
        assert (a != b).mean() > 0.95 * (0.75 if a.shape[1] == 4 else 1.0)


# ------------------------------------------------------------------------------------------------ statistics
def _series(p, ticks, R=64, W=16, seed=0):
    """(ticks, N, 3) errors and (ticks, N, 4) believed gs of a run without resets after the first call"""
    cfg = _cfg(R, W)
    N = R * W
    hs = HostState(cfg)
    pose, goal, gs = _inputs(np.random.default_rng(seed), N)
    none = np.zeros((N, 4), np.uint8)
    errs, outs = [], []
    for t in range(ticks):
        outs.append(observe_host(cfg, p, hs, t, pose, goal, gs, None if t == 0 else none))
        errs.append(hs.err[:, 0:3].copy())
    return np.stack(errs), np.stack(outs), gs


@pytest.mark.parametrize('tau', [0.0, 0.5, 2.0])
def test_stationary_deviation_and_autocorrelation(built, tau):
    """~1.2e5 agent-ticks: each component's standard deviation within 3 % of sigma at every tick's spread, and the lag-1
    autocorrelation within 0.02 of rho"""
    p = LocalizationParams(pose_sigma=(0.2, 0.2), heading_sigma=(0.1, 0.1), correlation_time=tau, seed=3)
    e, _, _ = _series(p, 120)
    rho = localization_ref.coefficients(tau, 0.1)[0]
    for k, sigma in ((0, 0.2), (1, 0.2), (2, 0.1)):
        x = e[:, :, k].astype(np.float64)
        assert abs(x.std() / sigma - 1) < 0.03, (k, x.std())
        assert abs(x.mean()) < 0.03 * sigma
        r = (x[1:] * x[:-1]).mean() / (x * x).mean()
        assert abs(r - float(rho)) < 0.02, (k, r, rho)


@pytest.mark.parametrize('lo,hi', [(0.05, 0.3), (0.0, 1.0)])
def test_sigmas_uniform_over_the_range(built, lo, hi):
    """102 400 per-episode draws of each sigma: KS test against uniform on [lo, hi]"""
    R, W = 64, 1600
    cfg = _cfg(R, W)
    p = LocalizationParams(pose_sigma=(lo, hi), heading_sigma=(lo, hi), seed=2024)
    hs = HostState(cfg)
    z = np.zeros((R * W, 4), np.float32)
    observe_host(cfg, p, hs, 9, z, z, z)
    for k in (0, 1):
        s = hs.sigma[:, k].astype(np.float64)
        assert s.min() >= lo and s.max() <= hi
        assert stats.kstest(s, 'uniform', args=(lo, hi - lo)).pvalue > 1e-3, k


def test_speed_noise_white_with_the_given_sigma(built):
    """~1.2e5 agent-ticks of speed noise: standard deviations within 3 %, no lag-1 correlation, no pose error"""
    p = LocalizationParams(speed_sigma=(0.05, 0.2), correlation_time=math.inf, seed=8)
    e, out, gs = _series(p, 120)
    assert not e.any()
    for k, sigma in ((2, 0.05), (3, 0.2)):
        d = out[:, :, k].astype(np.float64) - gs[None, :, k]
        assert abs(d.std() / sigma - 1) < 0.03 and abs(d.mean()) < 0.03 * sigma
        assert abs((d[1:] * d[:-1]).mean() / (d * d).mean()) < 0.02


# ------------------------------------------------------------------------------------------------ arguments
def _struct(**kw):
    d = dict(xy_lo=0.1, xy_hi=0.2, theta_lo=0.0, theta_hi=0.0, tau=2.0, v_sigma=0.0, w_sigma=0.0, seed=0,
             stream_id=0)
    d.update(kw)
    return _lib.LocalizationParams(d['xy_lo'], d['xy_hi'], d['theta_lo'], d['theta_hi'], d['tau'], d['v_sigma'],
                                   d['w_sigma'], d['seed'], d['stream_id'])


def _buffers(N=8):
    err, sigma = np.zeros((N, 4), np.float32), np.zeros((N, 2), np.float32)
    pose, goal = np.ones((N, 4), np.float32), np.full((N, 4), 2.0, np.float32)
    gs_in, gs_out = np.full((N, 4), 0.5, np.float32), np.zeros((N, 4), np.float32)
    return err, sigma, pose, goal, gs_in, gs_out


def _calls(lib, cfg, p, err, sigma, pose, goal, gs_in, gs_out, null=None):
    """both entries with the buffers given; `null` names one pointer passed as NULL.  The device entry never reaches a
    launch when an argument is invalid."""
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    st = _lib.LocalizationState(None if null == 'err' else err.ctypes.data,
                                None if null == 'sigma' else sigma.ctypes.data)
    env = _lib.EnvState(None if null == 'pose' else pose.ctypes.data, None if null == 'goal' else goal.ctypes.data,
                        None, None)
    a = dict(cfg=cfg, p=C.byref(p), st=C.byref(st), env=C.byref(env), gin=vp(gs_in), gout=vp(gs_out))
    for k in ('cfg', 'p', 'st', 'env', 'gin', 'gout'):
        if null == k:
            a[k] = None
    return [lib.rlca_localization_observe(a['cfg'], a['p'], a['st'], 0, None, a['env'], a['gin'], a['gout'], None),
            lib.rlca_localization_observe_host(a['cfg'], a['p'], a['st'], 0, None, a['env'], a['gin'], a['gout'])]


BAD_PARAMS = [dict(xy_lo=-0.1), dict(xy_lo=0.3, xy_hi=0.2), dict(xy_hi=math.inf), dict(xy_lo=math.nan),
              dict(xy_hi=math.nan), dict(theta_lo=-1.0, theta_hi=0.0), dict(theta_lo=0.2, theta_hi=0.1),
              dict(theta_hi=math.inf), dict(theta_lo=math.nan, theta_hi=math.nan), dict(tau=-1.0),
              dict(tau=-math.inf), dict(tau=math.nan), dict(v_sigma=-0.1), dict(v_sigma=math.inf),
              dict(w_sigma=math.nan), dict(w_sigma=-1e-30), dict(stream_id=1 << 24)]


@pytest.mark.parametrize('bad', BAD_PARAMS, ids=lambda d: ','.join('%s=%r' % kv for kv in d.items()))
def test_invalid_params_rejected(built, bad):
    lib = _lib.load()
    cfg = _cfg(4, 2)
    bufs = _buffers()
    keep = [b.copy() for b in bufs]
    assert _calls(lib, C.byref(cfg), _struct(**bad), *bufs) == [1, 1]
    assert b'localization' in lib.rlca_last_error()
    assert all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(bufs, keep))


@pytest.mark.parametrize('field,value', [('robots_per_world', 0), ('robots_per_world', 65), ('num_worlds', 0),
                                         ('world_offset', -1)])
def test_invalid_config_rejected(built, field, value):
    lib = _lib.load()
    cfg = _cfg(4, 2)
    setattr(cfg, field, value)
    assert _calls(lib, C.byref(cfg), _struct(), *_buffers()) == [1, 1]


@pytest.mark.parametrize('null', ['cfg', 'p', 'st', 'err', 'sigma', 'env', 'pose', 'goal', 'gin', 'gout'])
def test_null_pointers_rejected(built, null):
    lib = _lib.load()
    cfg = _cfg(4, 2)
    assert _calls(lib, C.byref(cfg), _struct(), *_buffers(), null=null) == [1, 1]


def test_edge_values_accepted(built):
    cfg = _cfg(64, 1)
    z = np.zeros((64, 4), np.float32)
    for kw in (dict(pose_sigma=(0.0, 0.0), correlation_time=0.0), dict(pose_sigma=(1e3, 1e3), heading_sigma=(7, 7)),
               dict(correlation_time=math.inf, speed_sigma=(0.0, 5.0)), dict(seed=2 ** 64 - 1)):
        out = observe_host(cfg, LocalizationParams(**kw), HostState(cfg), 2 ** 32 - 1, z, z, z,
                           stream_id=(1 << 24) - 1)
        assert np.isfinite(out).all()


@pytest.mark.parametrize('kw', [dict(pose_sigma=(-0.1, 0.1)), dict(pose_sigma=(0.3, 0.2)),
                                dict(pose_sigma=(0.1, math.inf)), dict(pose_sigma=(math.nan, 0.1)),
                                dict(heading_sigma=(0.2, 0.1)), dict(heading_sigma=0.1),
                                dict(heading_sigma=(0.1, 0.2, 0.3)), dict(heading_sigma=(True, 0.2)),
                                dict(pose_sigma=('a', 0.1)), dict(speed_sigma=(-0.1, 0.1)),
                                dict(speed_sigma=(0.1, math.nan)), dict(speed_sigma=(0.1, math.inf)),
                                dict(correlation_time=-1.0), dict(correlation_time=math.nan),
                                dict(correlation_time=-math.inf), dict(correlation_time='2'),
                                dict(correlation_time=True), dict(pose_sigma=(0.0, 1e39)),
                                dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.5)])
def test_localization_params_validated(kw):
    with pytest.raises(ValueError):
        LocalizationParams(**kw)


def test_localization_params_hold_float32():
    p = LocalizationParams(pose_sigma=(0.1, 0.3), heading_sigma=(0, 0), speed_sigma=(0.05, 0.1), seed=3)
    assert p.pose_sigma == (float(np.float32(0.1)), float(np.float32(0.3))) and p.heading_sigma == (0.0, 0.0)
    assert p.correlation_time == 2.0 and LocalizationParams(correlation_time=math.inf).correlation_time == math.inf
    assert p.speed_sigma == (float(np.float32(0.05)), float(np.float32(0.1)))
    assert p.on and not LocalizationParams().on and LocalizationParams(speed_sigma=(0, 0.1)).on
    assert p.as_dict() == {'pose_sigma': list(p.pose_sigma), 'heading_sigma': [0.0, 0.0], 'correlation_time': 2.0,
                           'speed_sigma': list(p.speed_sigma), 'seed': 3}


def test_localization_stream_id_validated():
    env = types.SimpleNamespace(N=4, device='cpu')
    for s in (-1, 1 << 24, 1.5):
        with pytest.raises(ValueError):
            Localization(env, LocalizationParams(pose_sigma=(0.1, 0.1)), stream_id=s)
    with pytest.raises(TypeError):
        Localization(env, {'pose_sigma': (0.1, 0.1)})


def test_zero_settings_allocate_nothing():
    env = types.SimpleNamespace(N=4, device='cpu')
    loc = Localization(env, LocalizationParams(correlation_time=0.0))
    assert loc.believed is None and loc._err is None and loc._sigma is None
    assert loc.errors.shape == (4, 3) and not loc.errors.any() and loc.sigmas.shape == (4, 2)


# ------------------------------------------------------------------------------------------------ command lines
POLICY = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')


@pytest.mark.parametrize('argv,msg', [
    (['--pose-error-time', '1'], '--pose-error-time applies'),
    (['--speed-error', '0.1', '--pose-error-time', '1'], '--pose-error-time applies'),
    (['--localization-seed', '3'], '--localization-seed applies'),
    (['--pose-error', '-0.1'], 'finite and >= 0'),
    (['--pose-error', '0.3,0.1'], 'lo <= hi'),
    (['--pose-error', 'inf'], 'finite and >= 0'),
    (['--heading-error', 'nan'], 'finite and >= 0'),
    (['--heading-error', '1,2,3'], '--heading-error'),
    (['--heading-error', 'x'], '--heading-error'),
    (['--speed-error', '0.1,-1'], 'finite and >= 0'),
    (['--pose-error', '0.1', '--pose-error-time', '-1'], 'correlation_time'),
    (['--pose-error', '0.1', '--pose-error-time', 'nan'], 'correlation_time'),
    (['--pose-error', '0.1', '--localization-seed', '-3'], 'localization seed'),
])
def test_evaluate_rejects_bad_localization_flags(built, capsys, argv, msg):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(['--scenario', 'stage2', '--policy', POLICY] + argv)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert msg in err, err


@pytest.mark.parametrize('who', [['--baseline', 'orca'], ['--baseline', 'nh-orca'], ['--policy', POLICY, '--hybrid']])
@pytest.mark.parametrize('flag', [['--pose-error', '0.1'], ['--heading-error', '0.05'], ['--speed-error', '0.1']])
def test_evaluate_refuses_localization_with_baselines_and_hybrid(built, capsys, who, flag):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(['--scenario', 'stage2'] + who + flag)
    assert e.value.code == 2
    assert 'read the true state' in capsys.readouterr().err


def test_localization_arguments(built):
    """the flags parse to LocalizationParams"""
    import argparse
    from rl_collision_avoidance_b200.localization import add_localization_arguments, localization_from_arguments
    ap = argparse.ArgumentParser()
    add_localization_arguments(ap)
    ap.add_argument('--seed', type=int, default=4)
    assert localization_from_arguments(ap, ap.parse_args([])) is None
    p = localization_from_arguments(ap, ap.parse_args(['--pose-error', '0.25']))
    assert (p.pose_sigma, p.heading_sigma, p.correlation_time, p.speed_sigma, p.seed) == \
        ((0.25, 0.25), (0.0, 0.0), 2.0, (0.0, 0.0), 4)
    p = localization_from_arguments(ap, ap.parse_args(['--pose-error', '0.125,0.5', '--heading-error', '0.25',
                                                       '--pose-error-time', 'inf', '--speed-error', '0.5,0.25',
                                                       '--localization-seed', '9']))
    assert (p.pose_sigma, p.heading_sigma, p.correlation_time, p.speed_sigma, p.seed) == \
        ((0.125, 0.5), (0.25, 0.25), math.inf, (0.5, 0.25), 9)
    p = localization_from_arguments(ap, ap.parse_args(['--speed-error', '0.25']))
    assert (p.pose_sigma, p.speed_sigma) == ((0.0, 0.0), (0.25, 0.25))
    p = localization_from_arguments(ap, ap.parse_args(['--heading-error', '0.1', '--pose-error-time', '0']))
    assert p.correlation_time == 0.0


@pytest.mark.parametrize('argv,msg', [
    (['--pose-error-time', '2'], '--pose-error-time applies'),
    (['--pose-error', '0.2,0.1'], 'lo <= hi'),
    (['--speed-error', 'a'], '--speed-error'),
    (['--localization-seed', '1'], '--localization-seed applies'),
    (['--mix', 'stage2:2,random:2', '--pose-error-time', '1'], '--pose-error-time applies'),
    (['--mix', 'stage2:2,random:2', '--heading-error', '-1'], 'finite and >= 0'),
])
def test_trainer_rejects_bad_localization_flags(built, capsys, argv, msg):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(argv=argv)
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


def test_kernel_does_not_spill(built, tmp_path):
    """-Xptxas -v of the file as build() compiles it: no spills and no stack frame"""
    import __graft_entry__ as g
    src = os.path.join(g.CSRC, 'rlca_localization.cu')
    cmd = [g.NVCC] + g.ARCH + g.COMMON + g.EXTRA['rlca_localization.cu'] + ['-Xptxas', '-v', '-c', src, '-o',
                                                                             str(tmp_path / 'loc.o')]
    err = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    blocks = re.findall(r"Function properties for (\w+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", err)
    assert len(blocks) == 1 and 'rlca_localization_kernel' in blocks[0][0], err
    assert tuple(int(x) for x in blocks[0][1:]) == (0, 0, 0), err
