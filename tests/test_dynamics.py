"""Acceleration limits without a GPU (DESIGN.md §9r): the host twin of csrc/rlca_dynamics.cu against the numpy
restatement (tests/dynamics_ref.py) over multi-tick sequences with random resets and crashes and commands that are NaN,
infinite, out of bounds or -0; the properties (limits in range and uniform, the exact ramp from rest, no step above
limit dt, non-binding limits as the identity of the tick's clip, independence of num_worlds and shards, streams and
seeds); every rejected argument at both ABI entries and in DynamicsParams, the command-line rules of evaluate.py and the
trainers, and the kernel's registers."""
import ctypes as C
import math
import os
import re
import subprocess
import types

import numpy as np
import pytest

import dynamics_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.dynamics import Dynamics, DynamicsParams, HostState, action_host
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(R=4, W=3, world_offset=0):
    cfg = fill_config(_lib.EnvConfig(), make_scenario('stage1'), num_worlds=W, beams=8, world_offset=world_offset)
    cfg.robots_per_world = R
    return cfg


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _bounds(cfg):
    return (cfg.v_min, cfg.v_max, cfg.w_min, cfg.w_max)


SPECIAL = np.array([np.nan, np.inf, -np.inf, -0.0, 3.2e38, -5.0, 7.0, 1e-30], np.float32)


def _commands(rng, N):
    """commands in and out of the bounds, with NaN, +-inf, -0 and finite values the tick treats as non-finite"""
    cmd = np.stack([rng.uniform(-0.5, 1.5, N), rng.uniform(-1.5, 1.5, N)], 1).astype(np.float32)
    hit = rng.random((N, 2)) < 0.1
    cmd[hit] = rng.choice(SPECIAL, int(hit.sum()))
    return cmd


def _run(R, W, p, ticks, seed=0, world_offset=0, stream=0, reset_p=0.1, crash_p=0.1):
    """ticks of the host twin and of the restatement side by side; asserts bit equality on every call"""
    cfg = _cfg(R, W, world_offset)
    N = R * W
    rng = np.random.default_rng(seed)
    hs = HostState(cfg)
    ref = dynamics_ref.Dynamics(R, W, p.linear, p.angular, p.seed, _bounds(cfg), cfg.dt, world_offset, stream)
    prev = None
    for t in range(ticks):
        cmd = _commands(rng, N)
        keep = cmd.copy()
        ex = action_host(cfg, p, hs, t, cmd, prev, stream_id=stream)
        assert np.array_equal(_bits(ex), _bits(ref.action(cmd, prev))), t
        assert np.array_equal(_bits(cmd), _bits(keep))
        assert np.array_equal(_bits(hs.vel), _bits(ex))
        assert np.array_equal(_bits(np.stack([hs.lin_limit, hs.ang_limit], 1)), _bits(ref.limit)), t
        prev = np.zeros((N, 4), np.uint8)
        prev[rng.random(N) < reset_p, 3] = 1
        prev[rng.random(N) < crash_p, 1] = 1
        prev[rng.random(N) < 0.1, 0] = 1            # done alone neither starts an episode nor stops the robot
    return hs


# ------------------------------------------------------------------------------------------------ reference
@pytest.mark.parametrize('linear,angular', [((2.0, 2.0), (0.0, 0.0)), ((0.0, 0.0), (3.0, 3.0)),
                                            ((0.5, 2.0), (1.0, 4.0)), ((1.0, 1.0), (2.0, 2.0)),
                                            ((0.3, 100.0), (0.1, 0.2)), ((0.0, 0.0), (0.0, 0.0))])
def test_host_twin_equals_restatement(built, linear, angular):
    p = DynamicsParams(linear=linear, angular=angular, seed=2 ** 40 + 3)
    hs = _run(5, 3, p, 50, seed=int(linear[1] * 10 + angular[1]), world_offset=7, stream=2)
    for (lo, hi), got in ((p.linear, hs.lin_limit), (p.angular, hs.ang_limit)):
        assert got.min() >= lo and got.max() <= hi


def test_host_twin_equals_restatement_many_resets_and_crashes(built):
    p = DynamicsParams(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=11)
    _run(8, 4, p, 60, seed=3, reset_p=0.4, crash_p=0.3)
    _run(8, 4, p, 40, seed=4, reset_p=0.0, crash_p=0.0)


# ------------------------------------------------------------------------------------------------ properties
@pytest.mark.parametrize('lo,hi', [(0.5, 2.0), (1.0, 4.0), (0.01, 100.0)])
def test_limits_uniform_over_the_range(built, lo, hi):
    """102 400 draws of each kind in [lo, hi]; 20 equal bins, each count within 5 sigma of uniform"""
    R, W = 64, 1600
    n = R * W
    cfg = _cfg(R, W)
    p = DynamicsParams(linear=(lo, hi), angular=(lo, hi), seed=2024)
    hs = HostState(cfg)
    action_host(cfg, p, hs, 9, np.zeros((n, 2), np.float32), None)
    k = 20
    for got in (hs.lin_limit, hs.ang_limit):
        assert got.min() >= np.float32(lo) and got.max() <= np.float32(hi)
        counts = np.histogram(got.astype(np.float64), bins=k, range=(p.linear[0], p.linear[1]))[0]
        sigma = math.sqrt(n * (1 / k) * (1 - 1 / k))
        assert (np.abs(counts - n / k) <= 5 * sigma).all(), counts
    assert np.array_equal(_bits(np.stack([hs.lin_limit, hs.ang_limit], 1)),
                          _bits(dynamics_ref.limits(2024, np.arange(n), 9, p.linear, p.angular)))
    assert not np.array_equal(hs.lin_limit, hs.ang_limit)          # the two words draw apart


def test_fixed_limits_ramp_from_rest_exactly(built):
    """a = 2 m/s^2 under a constant v = 1: 0.2, 0.4, 0.6, 0.8, then 1.0 itself; b = 4 rad/s^2 under w = -1: -0.4, -0.8,
    -1.0; a crash restarts from rest, a reset too"""
    R, W = 2, 2
    N = R * W
    cfg = _cfg(R, W)
    p = DynamicsParams(linear=(2.0, 2.0), angular=(4.0, 4.0), seed=1)
    hs = HostState(cfg)
    cmd = np.tile(np.float32([1.0, -1.0]), (N, 1))
    s_v, s_w = np.float32(2.0) * np.float32(cfg.dt), np.float32(4.0) * np.float32(cfg.dt)
    v, w = [], []
    flags = None
    for t in range(7):
        ex = action_host(cfg, p, hs, t, cmd, flags)
        v.append(ex[:, 0].copy())
        w.append(ex[:, 1].copy())
        flags = np.zeros((N, 4), np.uint8)
    want_v = [s_v, s_v + s_v, s_v + s_v + s_v, s_v + s_v + s_v + s_v, 1.0, 1.0, 1.0]
    want_w = [-s_w, -s_w - s_w, -1.0, -1.0, -1.0, -1.0, -1.0]
    for t in range(7):
        assert np.array_equal(_bits(v[t]), _bits(np.full(N, want_v[t], np.float32))), t
        assert np.array_equal(_bits(w[t]), _bits(np.full(N, want_w[t], np.float32))), t
    flags[0, 1] = 1                                  # robot 0 crashed, robot 1 re-spawned on the tick before
    flags[1, 3] = 1
    ex = action_host(cfg, p, hs, 7, cmd, flags)
    assert np.array_equal(_bits(ex[:2]), _bits(np.float32([[s_v, -s_w], [s_v, -s_w]])))
    assert np.array_equal(_bits(ex[2:]), _bits(np.float32([[1.0, -1.0], [1.0, -1.0]])))


@pytest.mark.parametrize('linear,angular', [((0.5, 2.0), (1.0, 4.0)), ((1.0, 1.0), (0.0, 0.0))])
def test_no_step_above_the_limit(built, linear, angular):
    """every tick |dv| <= a dt and |dw| <= b dt (up to the rounding of prev + s), except on fresh and crashed rows,
    which start from rest"""
    R, W = 6, 5
    N = R * W
    cfg = _cfg(R, W)
    p = DynamicsParams(linear=linear, angular=angular, seed=8)
    hs = HostState(cfg)
    rng = np.random.default_rng(1)
    prev_ex, flags = None, None
    for t in range(60):
        ex = action_host(cfg, p, hs, t, _commands(rng, N), flags)
        lim = np.stack([hs.lin_limit, hs.ang_limit], 1) * np.float32(cfg.dt)
        base = np.zeros_like(ex) if prev_ex is None else prev_ex.copy()
        if flags is not None:
            base[(flags[:, 3] != 0) | (flags[:, 1] != 0)] = 0.0
        step = np.abs(ex.astype(np.float64) - base)
        ulp = np.spacing(np.maximum(np.abs(ex), np.abs(base)).astype(np.float32)).astype(np.float64)
        for k, on in ((0, p.linear_on), (1, p.angular_on)):
            if on:                                   # prev + s rounds to the nearest float: half an ulp of slack
                assert (step[:, k] <= lim[:, k] + ulp[:, k] / 2).all(), t
        assert (ex[:, 0] >= cfg.v_min).all() and (ex[:, 0] <= cfg.v_max).all()
        assert (ex[:, 1] >= cfg.w_min).all() and (ex[:, 1] <= cfg.w_max).all()
        prev_ex = ex
        flags = np.zeros((N, 4), np.uint8)
        flags[rng.random(N) < 0.05, 3] = 1
        flags[rng.random(N) < 0.05, 1] = 1


def test_non_binding_limits_give_the_ticks_command(built):
    """a >= (v_max - v_min) / dt and b >= (w_max - w_min) / dt never bind: the output is the sanitised, clipped
    command bit for bit, whatever the state; both kinds off give the same"""
    R, W = 8, 4
    N = R * W
    cfg = _cfg(R, W)
    rng = np.random.default_rng(5)
    for p in (DynamicsParams(linear=(10.0, 10.0), angular=(20.0, 20.0), seed=3),
              DynamicsParams(linear=(10.0, 100.0), angular=(20.0, 50.0), seed=4), DynamicsParams(seed=5)):
        hs = HostState(cfg)
        flags = None
        for t in range(40):
            cmd = _commands(rng, N)
            ex = action_host(cfg, p, hs, t, cmd, flags)
            want = np.stack([dynamics_ref.target(cmd[:, 0], cfg.v_min, cfg.v_max),
                             dynamics_ref.target(cmd[:, 1], cfg.w_min, cfg.w_max)], 1)
            assert np.array_equal(_bits(ex), _bits(want)), (p, t)
            flags = np.zeros((N, 4), np.uint8)
            flags[rng.random(N) < 0.1, 3] = 1
    # the restatement's target is the tick's rule: NaN, +-inf and |x| > 3e38 give 0, -0 passes, the rest clip
    got = dynamics_ref.target(SPECIAL, 0.0, 1.0)
    assert np.array_equal(_bits(got), _bits(np.float32([0, 0, 0, -0.0, 0, 0, 1, 1e-30])))


def test_limits_independent_of_num_worlds_and_shards(built):
    R = 6
    p = DynamicsParams(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=77)

    def draws(W, off):
        cfg = _cfg(R, W, world_offset=off)
        hs = HostState(cfg)
        action_host(cfg, p, hs, 4, np.zeros((R * W, 2), np.float32), None, stream_id=1)
        return np.stack([hs.lin_limit, hs.ang_limit], 1)

    full = draws(200, 0)
    assert np.array_equal(_bits(draws(3, 0)), _bits(full[:3 * R]))
    for off, cnt in ((0, 70), (70, 1), (71, 129)):
        assert np.array_equal(_bits(draws(cnt, off)), _bits(full[off * R:(off + cnt) * R]))


@pytest.mark.parametrize('change', ['stream', 'seed', 'seed_hi', 'draw'])
def test_other_stream_seed_or_draw_gives_other_limits(built, change):
    R, W = 16, 8
    N = R * W
    cfg = _cfg(R, W)
    base = dict(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=1)
    other, stream, draw = dict(base), 0, 0
    if change == 'stream':
        stream = 1
    elif change == 'seed':
        other['seed'] = 2
    elif change == 'seed_hi':
        other['seed'] = 1 + (1 << 32)
    else:
        draw = 1
    out = []
    for kw, s, d in ((base, 0, 0), (other, stream, draw)):
        hs = HostState(cfg)
        action_host(cfg, DynamicsParams(**kw), hs, d, np.zeros((N, 2), np.float32), None, stream_id=s)
        out.append((hs.lin_limit.copy(), hs.ang_limit.copy()))
    for k in (0, 1):
        assert (out[0][k] != out[1][k]).mean() > 0.95


# ------------------------------------------------------------------------------------------------ arguments
def _struct(**kw):
    d = dict(lin_lo=1.0, lin_hi=2.0, ang_lo=0.0, ang_hi=0.0, seed=0, stream_id=0)
    d.update(kw)
    return _lib.DynamicsParams(d['lin_lo'], d['lin_hi'], d['ang_lo'], d['ang_hi'], d['seed'], d['stream_id'])


def _state(N=8):
    bufs = (np.zeros((N, 2), np.float32), np.zeros(N, np.float32), np.zeros(N, np.float32))
    return bufs, _lib.DynamicsState(*(b.ctypes.data for b in bufs))


def _entries(lib, cfg, p, st, cin, cout):
    """both entries called with valid buffers; the device entry never reaches a launch when an argument is invalid"""
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    return {'device': lambda: lib.rlca_dynamics_action(cfg, p, st, 0, None, vp(cin), vp(cout), None),
            'host': lambda: lib.rlca_dynamics_action_host(cfg, p, st, 0, None, vp(cin), vp(cout))}


BAD_PARAMS = [dict(lin_lo=0.0), dict(lin_lo=-1.0), dict(lin_lo=3.0, lin_hi=2.0), dict(lin_hi=100.5),
              dict(lin_lo=math.nan), dict(lin_hi=math.inf), dict(lin_lo=math.inf, lin_hi=math.inf),
              dict(ang_lo=0.0, ang_hi=1.0), dict(ang_lo=1.0, ang_hi=0.0), dict(ang_lo=-1.0, ang_hi=-1.0),
              dict(ang_lo=math.nan, ang_hi=math.nan), dict(ang_lo=2.0, ang_hi=math.nan),
              dict(stream_id=1 << 24)]


@pytest.mark.parametrize('bad', BAD_PARAMS, ids=lambda d: ','.join('%s=%r' % kv for kv in d.items()))
def test_invalid_params_rejected(built, bad):
    lib = _lib.load()
    cfg = _cfg(4, 2)
    bufs, st = _state()
    cin, cout = np.full((8, 2), 0.5, np.float32), np.zeros((8, 2), np.float32)
    keep = cin.copy()
    for name, call in _entries(lib, C.byref(cfg), C.byref(_struct(**bad)), C.byref(st), cin, cout).items():
        assert call() == 1, name
        assert b'dynamics' in lib.rlca_last_error()
    assert np.array_equal(_bits(cin), _bits(keep)) and not cout.any()
    assert not any(b.any() for b in bufs)


@pytest.mark.parametrize('field,value', [('robots_per_world', 0), ('robots_per_world', 65), ('num_worlds', 0),
                                         ('world_offset', -1)])
def test_invalid_config_rejected(built, field, value):
    lib = _lib.load()
    cfg = _cfg(4, 2)
    setattr(cfg, field, value)
    _, st = _state()
    cin, cout = np.full((8, 2), 0.5, np.float32), np.zeros((8, 2), np.float32)
    for name, call in _entries(lib, C.byref(cfg), C.byref(_struct()), C.byref(st), cin, cout).items():
        assert call() == 1, name


def test_null_pointers_rejected(built):
    lib = _lib.load()
    cfg, p = _cfg(4, 2), _struct()
    bufs, st = _state()
    buf = np.zeros((8, 2), np.float32)
    vp = buf.ctypes.data_as(C.c_void_p)
    c, pp, s = C.byref(cfg), C.byref(p), C.byref(st)
    calls = [lib.rlca_dynamics_action(None, pp, s, 0, None, vp, vp, None),
             lib.rlca_dynamics_action(c, None, s, 0, None, vp, vp, None),
             lib.rlca_dynamics_action(c, pp, None, 0, None, vp, vp, None),
             lib.rlca_dynamics_action(c, pp, s, 0, None, None, vp, None),
             lib.rlca_dynamics_action(c, pp, s, 0, None, vp, None, None),
             lib.rlca_dynamics_action_host(None, pp, s, 0, None, vp, vp),
             lib.rlca_dynamics_action_host(c, None, s, 0, None, vp, vp),
             lib.rlca_dynamics_action_host(c, pp, None, 0, None, vp, vp),
             lib.rlca_dynamics_action_host(c, pp, s, 0, None, None, vp),
             lib.rlca_dynamics_action_host(c, pp, s, 0, None, vp, None)]
    for k in range(3):                               # every state buffer, whichever kind is on
        ptrs = [b.ctypes.data for b in bufs]
        ptrs[k] = None
        s2 = C.byref(_lib.DynamicsState(*ptrs))
        calls += [lib.rlca_dynamics_action(c, pp, s2, 0, None, vp, vp, None),
                  lib.rlca_dynamics_action_host(c, pp, s2, 0, None, vp, vp)]
    assert calls == [1] * len(calls)


def test_edge_values_accepted(built):
    cfg = _cfg(64, 1)
    for kw in (dict(linear=(100.0, 100.0), angular=(100.0, 100.0)), dict(linear=(1e-6, 100.0)),
               dict(angular=(0.25, 0.25), seed=2 ** 64 - 1), dict()):
        p = DynamicsParams(**kw)
        ex = action_host(cfg, p, HostState(cfg), 2 ** 32 - 1, np.full((64, 2), 0.5, np.float32), None,
                         stream_id=(1 << 24) - 1)
        assert np.isfinite(ex).all()


@pytest.mark.parametrize('kw', [dict(linear=(0.0, 1.0)), dict(linear=(-1.0, 1.0)), dict(linear=(2.0, 1.0)),
                                dict(linear=(1.0, 100.5)), dict(linear=(math.nan, 1.0)), dict(linear=(1.0, math.inf)),
                                dict(angular=(1.0, 0.0)), dict(angular=(1e-46, 1.0)), dict(angular=3.0),
                                dict(angular=(1.0, 2.0, 3.0)), dict(angular=(True, 2.0)), dict(linear=('a', 1.0)),
                                dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.5)])
def test_dynamics_params_validated(kw):
    with pytest.raises(ValueError):
        DynamicsParams(**kw)


def test_dynamics_params_hold_float32():
    p = DynamicsParams(linear=(0.3, 1.7), angular=(2, 2), seed=3)
    assert p.linear == (float(np.float32(0.3)), float(np.float32(1.7))) and p.angular == (2.0, 2.0)
    assert p.linear_on and p.angular_on and not DynamicsParams().linear_on
    assert p.as_dict() == {'linear': list(p.linear), 'angular': [2.0, 2.0], 'seed': 3}


def test_dynamics_stream_id_validated():
    env = types.SimpleNamespace(N=4, device='cpu')
    for s in (-1, 1 << 24, 1.5):
        with pytest.raises(ValueError):
            Dynamics(env, DynamicsParams(linear=(1, 1)), stream_id=s)
    with pytest.raises(TypeError):
        Dynamics(env, {'linear': (1, 1)})


# ------------------------------------------------------------------------------------------------ command lines
POLICY = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')


@pytest.mark.parametrize('argv,msg', [
    (['--accel-limit', '0'], '--accel-limit: a limit must be > 0'),
    (['--accel-limit', '-1'], '--accel-limit: a limit must be > 0'),
    (['--accel-limit', '101'], '0 < lo <= hi <= 100'),
    (['--accel-limit', '2,1'], '0 < lo <= hi <= 100'),
    (['--accel-limit', 'nan'], '0 < lo <= hi <= 100'),
    (['--angular-accel-limit', 'inf'], '0 < lo <= hi <= 100'),
    (['--angular-accel-limit', '1,2,3'], '--angular-accel-limit'),
    (['--angular-accel-limit', 'x'], '--angular-accel-limit'),
    (['--dynamics-seed', '3'], '--dynamics-seed applies'),
    (['--accel-limit', '1', '--dynamics-seed', '-3'], 'dynamics seed'),
])
def test_evaluate_rejects_bad_dynamics_flags(built, capsys, argv, msg):
    import evaluate
    for who in (['--policy', POLICY], ['--baseline', 'nh-orca']):
        with pytest.raises(SystemExit) as e:
            evaluate.main(['--scenario', 'stage2'] + who + argv)
        assert e.value.code == 2
        err = capsys.readouterr().err
        assert msg in err, err


def test_dynamics_arguments(built):
    """the flags parse to DynamicsParams"""
    import argparse
    from rl_collision_avoidance_b200.dynamics import add_dynamics_arguments, dynamics_from_arguments
    ap = argparse.ArgumentParser()
    add_dynamics_arguments(ap)
    ap.add_argument('--seed', type=int, default=4)
    assert dynamics_from_arguments(ap, ap.parse_args([])) is None
    p = dynamics_from_arguments(ap, ap.parse_args(['--accel-limit', '2']))
    assert (p.linear, p.angular, p.seed, p.linear_on, p.angular_on) == ((2.0, 2.0), (0.0, 0.0), 4, True, False)
    p = dynamics_from_arguments(ap, ap.parse_args(['--accel-limit', '0.5,2', '--angular-accel-limit', '1,4',
                                                   '--dynamics-seed', '9']))
    assert (p.linear, p.angular, p.seed) == ((0.5, 2.0), (1.0, 4.0), 9)
    p = dynamics_from_arguments(ap, ap.parse_args(['--angular-accel-limit', '3']))
    assert (p.linear, p.angular) == ((0.0, 0.0), (3.0, 3.0))


@pytest.mark.parametrize('argv,msg', [
    (['--accel-limit', '0'], 'a limit must be > 0'),
    (['--angular-accel-limit', '2,1'], '0 < lo <= hi <= 100'),
    (['--accel-limit', 'a'], '--accel-limit'),
    (['--dynamics-seed', '1'], '--dynamics-seed applies'),
])
def test_trainer_rejects_bad_dynamics_flags(built, capsys, argv, msg):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(argv=argv)
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


def test_kernel_does_not_spill(built, tmp_path):
    """-Xptxas -v of the file as build() compiles it: no spills and no stack frame"""
    import __graft_entry__ as g
    src = os.path.join(g.CSRC, 'rlca_dynamics.cu')
    cmd = [g.NVCC] + g.ARCH + g.COMMON + g.EXTRA['rlca_dynamics.cu'] + ['-Xptxas', '-v', '-c', src, '-o',
                                                                         str(tmp_path / 'dyn.o')]
    err = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    blocks = re.findall(r"Function properties for (\w+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", err)
    assert len(blocks) == 1 and 'rlca_dynamics_action_kernel' in blocks[0][0], err
    assert tuple(int(x) for x in blocks[0][1:]) == (0, 0, 0), err
