"""Sensing and command latency without a GPU (DESIGN.md §9q): the host twins of csrc/rlca_latency.cu against the numpy
restatement (tests/latency_ref.py) over multi-tick sequences with random resets, their properties (delays in range and
uniform, the delayed frame and command, zero settings as the identity with nothing allocated, independence of
num_worlds and shards, streams and seeds), every rejected argument at the four ABI entries and in LatencyParams, the
command-line rules of evaluate.py and the trainers, and the kernels' registers."""
import ctypes as C
import math
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

import latency_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.latency import HostState, Latency, LatencyParams, action_host, scan_host
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(R=4, W=3, B=16, world_offset=0):
    cfg = fill_config(_lib.EnvConfig(), make_scenario('stage1'), num_worlds=W, beams=B, world_offset=world_offset)
    cfg.robots_per_world = R
    return cfg


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _frames(rng, N, B):
    return (rng.uniform(0.05, 5.95, (N, B)) / 6.0 - 0.5).astype(np.float32)


def _tick_stack(stack, newest, flags):
    """what the tick writes into stack_out: the FIFO shifted by one, three copies for re-spawned rows"""
    out = np.empty_like(stack)
    out[:, 0:2] = stack[:, 1:3]
    out[:, 2] = newest
    fresh = flags[:, 3] != 0
    out[fresh, 0] = newest[fresh]
    out[fresh, 1] = newest[fresh]
    return out


def _run(R, W, B, p, ticks, seed=0, world_offset=0, stream=0, reset_p=0.1):
    """ticks of the host twins and of the restatement side by side; asserts bit equality on every call"""
    cfg = _cfg(R, W, B, world_offset)
    N = R * W
    rng = np.random.default_rng(seed)
    hs = HostState(cfg, p)
    ref = latency_ref.Latency(R, W, p.scan_delay, p.command_delay, p.seed, world_offset, stream)
    first = _frames(rng, N, B)
    st = np.repeat(first[:, None], 3, 1)
    st_ref = st.copy()
    scan_host(cfg, p, hs, 0, st, None, stream_id=stream)
    ref.scan(st_ref, None)
    assert np.array_equal(_bits(st), _bits(st_ref))
    prev = None
    for t in range(ticks):
        cmd = np.stack([rng.uniform(-0.2, 1.2, N), rng.uniform(-1.2, 1.2, N)], 1).astype(np.float32)
        ex = action_host(cfg, p, hs, t, cmd, prev, stream_id=stream)
        assert np.array_equal(_bits(ex), _bits(ref.action(cmd, prev))), t
        flags = np.zeros((N, 4), np.uint8)
        flags[rng.random(N) < reset_p, 3] = 1
        flags[rng.random(N) < 0.1, 0] = 1           # done alone does not start an episode
        newest = _frames(rng, N, B)
        st = _tick_stack(st, newest, flags)
        st_ref = st.copy()
        scan_host(cfg, p, hs, t + 1, st, flags, stream_id=stream)
        ref.scan(st_ref, flags)
        assert np.array_equal(_bits(st), _bits(st_ref)), t
        if p.scan_on:
            assert np.array_equal(hs.scan_delay, ref.d)
        if p.command_on:
            assert np.array_equal(hs.cmd_delay, ref.l)
        prev = flags
    return hs


# ------------------------------------------------------------------------------------------------ reference
@pytest.mark.parametrize('B', [16, 13, 4])
@pytest.mark.parametrize('scan,cmd', [((2, 2), (0, 0)), ((0, 0), (3, 3)), ((0, 4), (1, 8)), ((8, 8), (0, 1)),
                                      ((1, 3), (2, 5))])
def test_host_twins_equal_restatement(built, B, scan, cmd):
    p = LatencyParams(scan_delay=scan, command_delay=cmd, seed=2 ** 40 + 3)
    hs = _run(5, 3, B, p, 40, seed=B, world_offset=7, stream=2)
    for (lo, hi), got in ((scan, hs.scan_delay), (cmd, hs.cmd_delay)):
        if hi > 0:
            assert got.min() >= lo and got.max() <= hi


def test_host_twins_equal_restatement_many_resets(built):
    p = LatencyParams(scan_delay=(0, 8), command_delay=(0, 8), seed=11)
    _run(8, 4, 8, p, 60, seed=3, reset_p=0.4)


# ------------------------------------------------------------------------------------------------ properties
@pytest.mark.parametrize('lo,hi', [(0, 4), (3, 8), (0, 1), (5, 5)])
def test_delays_uniform_over_the_range(built, lo, hi):
    """>= 10^5 draws of each kind: every value of [lo, hi] drawn, each count within 5 sigma of uniform"""
    R, W = 64, 1600
    n = R * W
    p = LatencyParams(scan_delay=(lo, hi), command_delay=(lo, hi), seed=2024)
    cfg = _cfg(R, W, 4)
    hs = HostState(cfg, p)
    scan_host(cfg, p, hs, 9, np.zeros((n, 3, 4), np.float32), None)
    action_host(cfg, p, hs, 9, np.zeros((n, 2), np.float32), None)
    k = hi - lo + 1
    for got in (hs.scan_delay, hs.cmd_delay):
        counts = np.bincount(got.astype(np.int64) - lo, minlength=k)
        assert counts.shape == (k,) and (counts > 0).all()
        sigma = math.sqrt(n * (1 / k) * (1 - 1 / k))
        assert (np.abs(counts - n / k) <= 5 * sigma + 1e-9).all(), counts
    assert np.array_equal(hs.scan_delay.astype(np.int64),
                          latency_ref.delays(2024, np.arange(n), 9, lo, hi, latency_ref.PURPOSE_SCAN))
    if hi > lo:
        assert not np.array_equal(hs.scan_delay, hs.cmd_delay)      # the two purposes draw apart


@pytest.mark.parametrize('d', [0, 1, 3, 8])
def test_fixed_scan_delay_delivers_the_frame_of_d_ticks_earlier(built, d):
    """lo = hi = d: after tick t the newest frame is the true frame of tick t - d, or the episode's first frame; the
    older frames are the frames delivered on the two calls before"""
    R, W, B = 3, 4, 8
    N = R * W
    cfg = _cfg(R, W, B)
    p = LatencyParams(scan_delay=(d, d), seed=5)
    hs = HostState(cfg, p)
    rng = np.random.default_rng(d)
    true = [_frames(rng, N, B)]                       # true[k]: the frame of call k (call 0: before the first tick)
    start = np.zeros(N, np.int64)
    st = np.repeat(true[0][:, None], 3, 1)
    scan_host(cfg, p, hs, 0, st, None)
    delivered = [st[:, 2].copy()]
    for k in range(1, 40):
        flags = np.zeros((N, 4), np.uint8)
        flags[rng.random(N) < 0.08, 3] = 1
        true.append(_frames(rng, N, B))
        st = _tick_stack(st, true[k], flags)
        scan_host(cfg, p, hs, k, st, flags)
        start[flags[:, 3] != 0] = k
        for a in range(N):
            src = max(k - d, start[a])
            assert np.array_equal(_bits(st[a, 2]), _bits(true[src][a])), (k, a)
            if flags[a, 3] == 0 and k >= 2 and start[a] <= k - 2:
                assert np.array_equal(_bits(st[a, 0:2]), _bits(np.stack([delivered[k - 2][a], delivered[k - 1][a]])))
        delivered.append(st[:, 2].copy())


@pytest.mark.parametrize('l', [0, 1, 2, 8])
def test_fixed_command_delay_executes_the_command_of_l_ticks_earlier(built, l):
    R, W = 4, 3
    N = R * W
    cfg = _cfg(R, W, 8)
    p = LatencyParams(command_delay=(l, l), seed=6)
    hs = HostState(cfg, p)
    rng = np.random.default_rng(l)
    issued = []
    start = np.zeros(N, np.int64)
    prev = None
    for t in range(40):
        cmd = np.stack([rng.uniform(0, 1, N), rng.uniform(-1, 1, N)], 1).astype(np.float32)
        issued.append(cmd)
        keep = cmd.copy()
        ex = action_host(cfg, p, hs, t, cmd, prev)
        assert np.array_equal(_bits(cmd), _bits(keep))
        if prev is not None:
            start[prev[:, 3] != 0] = t
        for a in range(N):
            want = issued[max(t - l, start[a])][a]         # l ticks earlier, or the episode's first command
            assert np.array_equal(_bits(ex[a]), _bits(want)), (t, a)
        prev = np.zeros((N, 4), np.uint8)
        prev[rng.random(N) < 0.1, 3] = 1


def test_zero_settings_are_the_identity_and_allocate_nothing(built):
    R, W, B = 4, 3, 13
    N = R * W
    cfg = _cfg(R, W, B)
    p = LatencyParams(seed=3)
    assert not p.scan_on and not p.command_on
    rng = np.random.default_rng(0)
    st = np.repeat(_frames(rng, N, B)[:, None], 3, 1)
    keep = st.copy()
    cmd = np.stack([rng.uniform(-1, 2, N), rng.uniform(-2, 2, N)], 1).astype(np.float32)
    cmd[0] = (-0.0, -0.0)
    hs = HostState(cfg, p)
    for t in range(3):
        scan_host(cfg, p, hs, t, st, np.ones((N, 4), np.uint8) if t else None)
        assert np.array_equal(_bits(st), _bits(keep))
        assert np.array_equal(_bits(action_host(cfg, p, hs, t, cmd)), _bits(cmd))
    # the C entries need no ring when a kind is off
    lib = _lib.load()
    null = _lib.LatencyState(None, None, None, None)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    out = np.empty_like(cmd)
    assert lib.rlca_latency_scan_host(C.byref(cfg), C.byref(p.struct()), C.byref(null), 0, None, vp(st)) == 0
    assert lib.rlca_latency_action_host(C.byref(cfg), C.byref(p.struct()), C.byref(null), 0, None, vp(cmd), vp(out)) == 0
    assert np.array_equal(_bits(out), _bits(cmd)) and np.array_equal(_bits(st), _bits(keep))
    # the Python object allocates nothing and returns what it was given
    env = types.SimpleNamespace(N=N, beam_mum=B, device='cpu')
    lat = Latency(env, p)
    assert lat._scan_ring is None and lat._cmd_ring is None and lat.executed is None
    ts, tc = torch.from_numpy(st.copy()), torch.from_numpy(cmd)
    assert lat.scan(ts) is ts and lat.action(tc) is tc
    assert lat.scan_calls == 1 and lat.action_calls == 1
    assert lat.scan_delays.tolist() == [0] * N and lat.command_delays.tolist() == [0] * N


def test_delays_independent_of_num_worlds_and_shards(built):
    R, B = 6, 8
    p = LatencyParams(scan_delay=(0, 8), command_delay=(1, 6), seed=77)

    def draws(W, off):
        cfg = _cfg(R, W, B, world_offset=off)
        hs = HostState(cfg, p)
        scan_host(cfg, p, hs, 4, np.zeros((R * W, 3, B), np.float32), None, stream_id=1)
        action_host(cfg, p, hs, 4, np.zeros((R * W, 2), np.float32), None, stream_id=1)
        return hs.scan_delay, hs.cmd_delay

    full = draws(200, 0)
    small = draws(3, 0)
    for f, s in zip(full, small):
        assert np.array_equal(s, f[:3 * R])
    for off, cnt in ((0, 70), (70, 1), (71, 129)):
        for f, s in zip(full, draws(cnt, off)):
            assert np.array_equal(s, f[off * R:(off + cnt) * R])


@pytest.mark.parametrize('change', ['stream', 'seed', 'seed_hi', 'draw'])
def test_other_stream_seed_or_draw_gives_other_delays(built, change):
    R, W, B = 16, 8, 4
    N = R * W
    cfg = _cfg(R, W, B)
    base = dict(scan_delay=(0, 8), command_delay=(0, 8), seed=1)
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
        p = LatencyParams(**kw)
        hs = HostState(cfg, p)
        scan_host(cfg, p, hs, d, np.zeros((N, 3, B), np.float32), None, stream_id=s)
        action_host(cfg, p, hs, d, np.zeros((N, 2), np.float32), None, stream_id=s)
        out.append((hs.scan_delay.copy(), hs.cmd_delay.copy()))
    for k in (0, 1):
        assert (out[0][k] != out[1][k]).mean() > 0.6


# ------------------------------------------------------------------------------------------------ arguments
def _struct(**kw):
    d = dict(scan_lo=1, scan_hi=2, cmd_lo=0, cmd_hi=3, seed=0, stream_id=0)
    d.update(kw)
    return _lib.LatencyParams(d['scan_lo'], d['scan_hi'], d['cmd_lo'], d['cmd_hi'], d['seed'], d['stream_id'])


def _state(N=8, B=8):
    bufs = (np.zeros((N, 9, B), np.float32), np.zeros((N, 9, 2), np.float32), np.zeros(N, np.uint8),
            np.zeros(N, np.uint8))
    return bufs, _lib.LatencyState(*(b.ctypes.data for b in bufs))


def _entries(lib, cfg, p, st, buf, buf2):
    """each entry called with valid buffers; the device entries never reach a launch when an argument is invalid"""
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    return {'scan': lambda: lib.rlca_latency_scan(cfg, p, st, 0, None, vp(buf), None),
            'action': lambda: lib.rlca_latency_action(cfg, p, st, 0, None, vp(buf2), vp(buf2), None),
            'scan_host': lambda: lib.rlca_latency_scan_host(cfg, p, st, 0, None, vp(buf)),
            'action_host': lambda: lib.rlca_latency_action_host(cfg, p, st, 0, None, vp(buf2), vp(buf2))}


BAD_PARAMS = [dict(scan_lo=-1), dict(cmd_lo=-1), dict(scan_lo=3, scan_hi=2), dict(cmd_lo=4, cmd_hi=3),
              dict(scan_hi=9), dict(cmd_hi=9), dict(scan_lo=9, scan_hi=9), dict(stream_id=1 << 24)]


@pytest.mark.parametrize('bad', BAD_PARAMS, ids=lambda d: ','.join('%s=%r' % kv for kv in d.items()))
def test_invalid_params_rejected(built, bad):
    lib = _lib.load()
    cfg = _cfg(4, 2, 8)
    bufs, st = _state()
    buf, buf2 = np.zeros((8, 3, 8), np.float32), np.full((8, 2), 0.5, np.float32)
    keep, keep2 = buf.copy(), buf2.copy()
    for name, call in _entries(lib, C.byref(cfg), C.byref(_struct(**bad)), C.byref(st), buf, buf2).items():
        assert call() == 1, name
        assert b'latency' in lib.rlca_last_error()
    assert np.array_equal(_bits(buf), _bits(keep)) and np.array_equal(_bits(buf2), _bits(keep2))
    assert not any(b.any() for b in bufs)


@pytest.mark.parametrize('field,value', [('robots_per_world', 0), ('robots_per_world', 65), ('num_worlds', 0),
                                         ('beams', 0), ('world_offset', -1)])
def test_invalid_config_rejected(built, field, value):
    lib = _lib.load()
    cfg = _cfg(4, 2, 8)
    setattr(cfg, field, value)
    _, st = _state()
    buf, buf2 = np.zeros((8, 3, 8), np.float32), np.full((8, 2), 0.5, np.float32)
    for name, call in _entries(lib, C.byref(cfg), C.byref(_struct()), C.byref(st), buf, buf2).items():
        assert call() == 1, name


def test_null_pointers_rejected(built):
    lib = _lib.load()
    cfg, p = _cfg(4, 2, 8), _struct()
    bufs, st = _state()
    buf = np.zeros((8, 3, 8), np.float32)
    vp = buf.ctypes.data_as(C.c_void_p)
    c, pp, s = C.byref(cfg), C.byref(p), C.byref(st)
    calls = [lib.rlca_latency_scan(None, pp, s, 0, None, vp, None),
             lib.rlca_latency_scan(c, None, s, 0, None, vp, None),
             lib.rlca_latency_scan(c, pp, None, 0, None, vp, None),
             lib.rlca_latency_scan(c, pp, s, 0, None, None, None),
             lib.rlca_latency_action(None, pp, s, 0, None, vp, vp, None),
             lib.rlca_latency_action(c, None, s, 0, None, vp, vp, None),
             lib.rlca_latency_action(c, pp, None, 0, None, vp, vp, None),
             lib.rlca_latency_action(c, pp, s, 0, None, None, vp, None),
             lib.rlca_latency_action(c, pp, s, 0, None, vp, None, None),
             lib.rlca_latency_scan_host(None, pp, s, 0, None, vp),
             lib.rlca_latency_scan_host(c, None, s, 0, None, vp),
             lib.rlca_latency_scan_host(c, pp, None, 0, None, vp),
             lib.rlca_latency_scan_host(c, pp, s, 0, None, None),
             lib.rlca_latency_action_host(None, pp, s, 0, None, vp, vp),
             lib.rlca_latency_action_host(c, None, s, 0, None, vp, vp),
             lib.rlca_latency_action_host(c, pp, None, 0, None, vp, vp),
             lib.rlca_latency_action_host(c, pp, s, 0, None, None, vp),
             lib.rlca_latency_action_host(c, pp, s, 0, None, vp, None)]
    assert calls == [1] * len(calls)
    # a kind that is on needs its ring and its delays
    for k in range(4):
        ptrs = [b.ctypes.data for b in bufs]
        ptrs[k] = None
        s2 = C.byref(_lib.LatencyState(*ptrs))
        scan_rc = lib.rlca_latency_scan_host(c, pp, s2, 0, None, vp)
        act_rc = lib.rlca_latency_action_host(c, pp, s2, 0, None, vp, vp)
        assert (scan_rc, act_rc) == ((1, 0) if k in (0, 2) else (0, 1)), k


def test_edge_values_accepted(built):
    cfg = _cfg(64, 1, 8)
    for kw in (dict(scan_delay=(8, 8), command_delay=(8, 8)), dict(scan_delay=(0, 8)), dict(seed=2 ** 64 - 1,
                                                                                           command_delay=(0, 1))):
        p = LatencyParams(**kw)
        hs = HostState(cfg, p)
        scan_host(cfg, p, hs, 2 ** 32 - 1, np.zeros((64, 3, 8), np.float32), None, stream_id=(1 << 24) - 1)
        action_host(cfg, p, hs, 2 ** 32 - 1, np.zeros((64, 2), np.float32), None, stream_id=(1 << 24) - 1)


@pytest.mark.parametrize('kw', [dict(scan_delay=(-1, 2)), dict(scan_delay=(3, 2)), dict(scan_delay=(0, 9)),
                                dict(command_delay=(0, 9)), dict(command_delay=(2, 1)), dict(command_delay=(1.5, 2)),
                                dict(command_delay=3), dict(scan_delay=(1, 2, 3)), dict(scan_delay=(True, 2)),
                                dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.5)])
def test_latency_params_validated(kw):
    with pytest.raises(ValueError):
        LatencyParams(**kw)


def test_latency_stream_id_validated():
    env = types.SimpleNamespace(N=4, beam_mum=8, device='cpu')
    for s in (-1, 1 << 24, 1.5):
        with pytest.raises(ValueError):
            Latency(env, LatencyParams(), stream_id=s)
    with pytest.raises(TypeError):
        Latency(env, {'scan_delay': (1, 1)})


# ------------------------------------------------------------------------------------------------ command lines
POLICY = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')


@pytest.mark.parametrize('argv,msg', [
    (['--baseline', 'orca', '--scan-delay', '2'], '--scan-delay applies to --policy only'),
    (['--baseline', 'nh-orca', '--scan-delay', '0,2'], '--scan-delay applies to --policy only'),
    (['--policy', POLICY, '--scan-delay', '-1'], '0 <= lo <= hi <= 8'),
    (['--policy', POLICY, '--scan-delay', '9'], '0 <= lo <= hi <= 8'),
    (['--policy', POLICY, '--command-delay', '3,1'], '0 <= lo <= hi <= 8'),
    (['--policy', POLICY, '--command-delay', '1,2,3'], '--command-delay'),
    (['--policy', POLICY, '--command-delay', '1.5'], '--command-delay'),
    (['--policy', POLICY, '--scan-delay', 'x'], '--scan-delay'),
    (['--policy', POLICY, '--latency-seed', '3'], '--latency-seed applies'),
    (['--policy', POLICY, '--scan-delay', '1', '--latency-seed', '-3'], 'latency seed'),
])
def test_evaluate_rejects_bad_latency_flags(built, capsys, argv, msg):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(['--scenario', 'stage2'] + argv)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert msg in err, err


def test_latency_arguments(built):
    """the flags parse to LatencyParams; --command-delay with a baseline parses (the run itself needs a GPU)"""
    import argparse
    from rl_collision_avoidance_b200.latency import add_latency_arguments, latency_from_arguments
    ap = argparse.ArgumentParser()
    add_latency_arguments(ap)
    ap.add_argument('--seed', type=int, default=4)
    assert latency_from_arguments(ap, ap.parse_args([])) is None
    p = latency_from_arguments(ap, ap.parse_args(['--command-delay', '2']))
    assert (p.scan_delay, p.command_delay, p.seed, p.scan_on, p.command_on) == ((0, 0), (2, 2), 4, False, True)
    p = latency_from_arguments(ap, ap.parse_args(['--scan-delay', '0,4', '--command-delay', '1,3', '--latency-seed',
                                                  '9']))
    assert (p.scan_delay, p.command_delay, p.seed) == ((0, 4), (1, 3), 9)
    assert p.as_dict() == {'scan_delay': [0, 4], 'command_delay': [1, 3], 'seed': 9}


@pytest.mark.parametrize('argv,msg', [
    (['--scan-delay', '9'], '0 <= lo <= hi <= 8'),
    (['--command-delay', '2,1'], '0 <= lo <= hi <= 8'),
    (['--command-delay', 'a'], '--command-delay'),
    (['--latency-seed', '1'], '--latency-seed applies'),
])
def test_trainer_rejects_bad_latency_flags(built, capsys, argv, msg):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(argv=argv)
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


def test_kernels_do_not_spill(built, tmp_path):
    """-Xptxas -v of the file as build() compiles it: no spills and no stack frame in any kernel"""
    import __graft_entry__ as g
    src = os.path.join(g.CSRC, 'rlca_latency.cu')
    cmd = [g.NVCC] + g.ARCH + g.COMMON + g.EXTRA['rlca_latency.cu'] + ['-Xptxas', '-v', '-c', src, '-o',
                                                                        str(tmp_path / 'lat.o')]
    err = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    blocks = re.findall(r"Function properties for (\w+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", err)
    names = [b[0] for b in blocks]
    for k in ('rlca_latency_scan_kernelILb0', 'rlca_latency_scan_kernelILb1', 'rlca_latency_action_kernel'):
        assert any(k in n for n in names), err
    assert len(blocks) == 3, err
    for name, stack, st, ld in blocks:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), (name, err)
