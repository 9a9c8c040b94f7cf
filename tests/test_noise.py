"""Sensor and actuation noise without a GPU (DESIGN.md §9p): the host twins of csrc/rlca_noise.cu against the numpy
restatement (tests/noise_ref.py), their properties (no-op at zero, dropout, no phantom returns, older frames, fresh
rows, bounds, zero commands, independence of num_worlds and shards, streams and seeds, the distribution), every rejected
argument at both ABI entries, the command-line rules of evaluate.py and the trainers, and the kernels' registers."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import noise_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.noise import NoiseParams, action_host, scan_host
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RMAX_O = np.float32(0.5)                 # the scan value of range_max, as the tick writes it


def _cfg(R=4, W=3, B=16, world_offset=0):
    cfg = fill_config(_lib.EnvConfig(), make_scenario('stage1'), num_worlds=W, beams=B, world_offset=world_offset)
    cfg.robots_per_world = R
    return cfg


def _stack(N, B, seed=0, no_return=0.1):
    """(N, 3, B) float32 normalised scans: ranges in [0.05, 5.95] m and a share of beams without a return"""
    rng = np.random.default_rng(seed)
    r = rng.uniform(0.05, 5.95, (N, 3, B))
    o = (r / 6.0 - 0.5).astype(np.float32)
    o[rng.random((N, 3, B)) < no_return] = RMAX_O
    return o


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _P(**kw):
    return NoiseParams(**kw)


# ------------------------------------------------------------------------------------------------ reference
@pytest.mark.parametrize('B', [16, 13, 512])
@pytest.mark.parametrize('draw,stream,seed', [(0, 0, 0), (7, 3, 2 ** 32 + 5), (2 ** 32 - 1, 2 ** 24 - 1, 2 ** 64 - 1)])
def test_dropout_decisions_exact(built, B, draw, stream, seed):
    R, W = 5, 3
    cfg = _cfg(R, W, B)
    p = _P(dropout=0.37, seed=seed)
    st = _stack(R * W, B)
    newest = st[:, 2].copy()
    scan_host(cfg, p, draw, st, np.zeros((R * W, 4), np.uint8), stream_id=stream)
    _, dropped, _, _ = noise_ref.scan(newest, dict(p.as_dict()), R, W, draw, stream=stream)
    assert np.array_equal(st[:, 2] == RMAX_O, dropped | (newest == RMAX_O))
    assert np.array_equal(_bits(st[:, 2][~dropped]), _bits(newest[~dropped]))    # sigma 0: the rest untouched
    assert 0 < dropped.sum() < dropped.size


@pytest.mark.parametrize('B', [16, 13, 512])
@pytest.mark.parametrize('sigma', [0.01, 0.1, 0.5, 3.0])
def test_range_noise_against_float64(built, B, sigma):
    R, W, draw, stream = 6, 4, 11, 2
    cfg = _cfg(R, W, B, world_offset=9)
    p = _P(range_sigma=sigma, dropout=0.2, seed=12345)
    st = _stack(R * W, B, seed=1)
    newest = st[:, 2].copy()
    scan_host(cfg, p, draw, st, np.zeros((R * W, 4), np.uint8), stream_id=stream)
    ref, dropped, z, rho = noise_ref.scan(newest, p.as_dict(), R, W, draw, world_offset=9, stream=stream)
    got = st[:, 2].astype(np.float64)
    assert np.array_equal(got[dropped], np.full(dropped.sum(), 0.5))
    err = np.abs(got - ref)
    tol = noise_ref.scan_tolerance(float(np.float32(sigma)), rho)
    ratio = (err / tol)[~dropped].max()
    assert ratio <= 1.0, ratio
    # and the rows really moved: a beam with a return, not dropped, changes by sigma |z|
    moved = ~dropped & (newest != RMAX_O)
    assert np.abs(got - newest)[moved].mean() > 0.1 * sigma / 6.0


@pytest.mark.parametrize('sigmas', [(0.1, 0.1), (0.3, 0.05), (2.0, 0.0), (0.0, 1.5)])
def test_action_noise_against_float64(built, sigmas):
    R, W, draw, stream = 8, 5, 3, 1
    cfg = _cfg(R, W, 8, world_offset=2)
    p = _P(v_gain_sigma=sigmas[0], w_gain_sigma=sigmas[1], seed=99)
    rng = np.random.default_rng(2)
    cmd = np.stack([rng.uniform(-0.2, 1.2, R * W), rng.uniform(-1.3, 1.3, R * W)], 1).astype(np.float32)
    got = action_host(cfg, p, draw, cmd, stream_id=stream).astype(np.float64)
    bounds = (cfg.v_min, cfg.v_max, cfg.w_min, cfg.w_max)
    ref, z, rho = noise_ref.action(cmd, p.as_dict(), bounds, R, W, draw, world_offset=2, stream=stream)
    s = np.array([np.float32(sigmas[0]), np.float32(sigmas[1])], np.float64)
    c = np.clip(cmd.astype(np.float64), [bounds[0], bounds[2]], [bounds[1], bounds[3]])
    tol = noise_ref.action_tolerance(c, s, rho[:, None])
    assert (np.abs(got - ref) <= tol).all(), np.abs(got - ref).max()


# ------------------------------------------------------------------------------------------------ properties
@pytest.mark.parametrize('B', [16, 13])
def test_zero_noise_is_bit_identity(built, B):
    R, W = 4, 3
    cfg = _cfg(R, W, B)
    p = _P(seed=5)
    st = _stack(R * W, B)
    ref = st.copy()
    flags = np.zeros((R * W, 4), np.uint8)
    scan_host(cfg, p, 1, st, flags)
    assert np.array_equal(_bits(st), _bits(ref))
    cmd = np.stack([np.linspace(0, 1, R * W), np.linspace(-1, 1, R * W)], 1).astype(np.float32)
    cmd[0] = (-0.0, -0.0)
    out = action_host(cfg, p, 1, cmd)
    assert np.array_equal(_bits(out), _bits(cmd))


def test_full_dropout_reads_range_max(built):
    R, W, B = 4, 2, 13
    st = _stack(R * W, B)
    older = st[:, :2].copy()
    scan_host(_cfg(R, W, B), _P(range_sigma=0.3, dropout=1.0, seed=3), 0, st, np.zeros((R * W, 4), np.uint8))
    assert (st[:, 2] == RMAX_O).all()
    assert np.array_equal(_bits(st[:, :2]), _bits(older))


def test_range_noise_never_makes_a_return(built):
    R, W, B = 4, 3, 64
    st = _stack(R * W, B, no_return=0.5)
    none = st[:, 2] == RMAX_O
    scan_host(_cfg(R, W, B), _P(range_sigma=5.0, seed=8), 0, st, np.zeros((R * W, 4), np.uint8))
    assert (st[:, 2][none] == RMAX_O).all()
    assert (st[:, 2] >= -0.5).all() and (st[:, 2] <= RMAX_O).all()
    # a large sigma clamps to [0, range_max]: both ends are reached
    assert (st[:, 2][~none] == np.float32(-0.5)).any() and (st[:, 2][~none] == RMAX_O).any()


@pytest.mark.parametrize('B', [16, 13])
def test_older_frames_untouched_and_fresh_rows_copied(built, B):
    R, W = 4, 3
    N = R * W
    st = _stack(N, B)
    before = st.copy()
    flags = np.zeros((N, 4), np.uint8)
    flags[::3, 3] = 1
    flags[1::3, 0] = 1                      # done alone does not make a row fresh
    scan_host(_cfg(R, W, B), _P(range_sigma=0.2, dropout=0.1, seed=4), 2, st, flags)
    fresh = flags[:, 3] != 0
    assert np.array_equal(_bits(st[~fresh, :2]), _bits(before[~fresh, :2]))
    for k in (0, 1):
        assert np.array_equal(_bits(st[fresh, k]), _bits(st[fresh, 2]))
    assert not np.array_equal(st[:, 2], before[:, 2])
    # no flags: every row fresh
    st2 = before.copy()
    scan_host(_cfg(R, W, B), _P(range_sigma=0.2, dropout=0.1, seed=4), 2, st2, None)
    assert np.array_equal(_bits(st2[:, 2]), _bits(st[:, 2]))
    assert np.array_equal(_bits(st2[:, 0]), _bits(st2[:, 2])) and np.array_equal(_bits(st2[:, 1]), _bits(st2[:, 2]))


def test_action_bounds_and_zero_commands(built):
    R, W = 16, 4
    cfg = _cfg(R, W, 8)
    N = R * W
    rng = np.random.default_rng(1)
    cmd = np.stack([rng.uniform(-1, 2, N), rng.uniform(-2, 2, N)], 1).astype(np.float32)
    cmd[:8, 0] = 0.0
    cmd[8:12, 0] = -0.0
    cmd[12:16, 1] = 0.0
    keep = cmd.copy()
    out = action_host(cfg, _P(v_gain_sigma=3.0, w_gain_sigma=3.0, seed=2), 0, cmd)
    assert np.array_equal(_bits(cmd), _bits(keep))                     # the command is not written
    assert (out[:, 0] >= cfg.v_min).all() and (out[:, 0] <= cfg.v_max).all()
    assert (out[:, 1] >= cfg.w_min).all() and (out[:, 1] <= cfg.w_max).all()
    assert np.array_equal(_bits(out[:12, 0]), _bits(cmd[:12, 0]))      # +0 and -0 stay as they are
    assert np.array_equal(_bits(out[12:16, 1]), _bits(cmd[12:16, 1]))
    # a gain never reverses a command
    c = np.clip(cmd, [cfg.v_min, cfg.w_min], [cfg.v_max, cfg.w_max])
    assert (out * c >= 0).all()


def test_draws_independent_of_num_worlds_and_shards(built):
    R, B = 6, 13
    p = _P(range_sigma=0.1, dropout=0.2, v_gain_sigma=0.1, w_gain_sigma=0.2, seed=77)
    big = _stack(200 * R, B)
    full = big.copy()
    flags = np.zeros((200 * R, 4), np.uint8)
    flags[::5, 3] = 1
    scan_host(_cfg(R, 200, B), p, 4, full, flags, stream_id=1)
    small = big[:3 * R].copy()
    scan_host(_cfg(R, 3, B), p, 4, small, flags[:3 * R], stream_id=1)
    assert np.array_equal(_bits(small), _bits(full[:3 * R]))
    for off, cnt in ((0, 70), (70, 1), (71, 129)):
        sh = big[off * R:(off + cnt) * R].copy()
        scan_host(_cfg(R, cnt, B, world_offset=off), p, 4, sh, flags[off * R:(off + cnt) * R], stream_id=1)
        assert np.array_equal(_bits(sh), _bits(full[off * R:(off + cnt) * R]))
    cmd = np.tile(np.float32([[0.5, 0.3]]), (200 * R, 1))
    a_full = action_host(_cfg(R, 200, B), p, 4, cmd, stream_id=1)
    a_sh = action_host(_cfg(R, 130, B, world_offset=70), p, 4, cmd[70 * R:], stream_id=1)
    assert np.array_equal(_bits(a_sh), _bits(a_full[70 * R:]))
    assert np.array_equal(_bits(action_host(_cfg(R, 3, B), p, 4, cmd[:3 * R], stream_id=1)), _bits(a_full[:3 * R]))


@pytest.mark.parametrize('change', ['stream', 'seed', 'draw', 'seed_hi'])
def test_other_stream_seed_or_draw_gives_other_draws(built, change):
    R, W, B = 4, 2, 64
    base = dict(range_sigma=0.1, dropout=0.3, v_gain_sigma=0.1, w_gain_sigma=0.1, seed=1)
    st0 = _stack(R * W, B)
    cmd = np.tile(np.float32([[0.5, 0.3]]), (R * W, 1))
    args = dict(draw=0, stream=0)
    other = dict(base)
    oargs = dict(args)
    if change == 'stream':
        oargs['stream'] = 2                 # 2 << 8 would overlap a purpose of the form 0x4E01
    elif change == 'seed':
        other['seed'] = 2
    elif change == 'seed_hi':
        other['seed'] = 1 + (1 << 32)
    else:
        oargs['draw'] = 1
    a, b = st0.copy(), st0.copy()
    scan_host(_cfg(R, W, B), _P(**base), args['draw'], a, None, stream_id=args['stream'])
    scan_host(_cfg(R, W, B), _P(**other), oargs['draw'], b, None, stream_id=oargs['stream'])
    diff = (a[:, 2] != b[:, 2]).mean()
    assert diff > 0.5, diff
    ca = action_host(_cfg(R, W, B), _P(**base), args['draw'], cmd, stream_id=args['stream'])
    cb = action_host(_cfg(R, W, B), _P(**other), oargs['draw'], cmd, stream_id=oargs['stream'])
    assert (ca != cb).all()


def test_distribution_over_a_million_beams(built):
    """z recovered from 10^6 perturbed beams at 3 m (no clamp within 30 sigma): |mean| < 5 / sqrt(n) and
    |std - 1| < 5 / sqrt(2 n), five standard errors; the dropout share within five standard errors of p."""
    R, W, B = 64, 31, 512
    n = R * W * B                            # 1 015 808 beams
    sigma = np.float32(0.1)
    st = np.zeros((R * W, 3, B), np.float32)  # o = 0 <=> r = 3 m
    scan_host(_cfg(R, W, B), _P(range_sigma=float(sigma), seed=2024), 5, st, None)
    r = (st[:, 2].astype(np.float64) + 0.5) * 6.0
    z = ((r - 3.0) / float(sigma)).ravel()
    assert abs(z.mean()) < 5 / math.sqrt(n), z.mean()
    assert abs(z.std() - 1.0) < 5 / math.sqrt(2 * n), z.std()
    assert abs(z.max()) < 7 and abs(z.min()) < 7
    st = np.zeros((R * W, 3, B), np.float32)
    scan_host(_cfg(R, W, B), _P(dropout=0.3, seed=2024), 5, st, None)
    share = (st[:, 2] == RMAX_O).mean()
    assert abs(share - 0.3) < 5 * math.sqrt(0.3 * 0.7 / n), share
    cmd = np.tile(np.float32([[0.5, 0.5]]), (R * W * 64, 1))
    out = action_host(_cfg(R, W * 64, B), _P(v_gain_sigma=0.1, w_gain_sigma=0.1, seed=1), 0, cmd)
    g = (out.astype(np.float64) / 0.5 - 1.0) / float(np.float32(0.1))
    m = g.shape[0]
    for k in (0, 1):
        assert abs(g[:, k].mean()) < 5 / math.sqrt(m) and abs(g[:, k].std() - 1.0) < 5 / math.sqrt(2 * m)
    assert abs(np.corrcoef(g[:, 0], g[:, 1])[0, 1]) < 5 / math.sqrt(m)


# ------------------------------------------------------------------------------------------------ arguments
def _bad_params():
    nan, inf = float('nan'), float('inf')
    out = []
    for k in ('range_sigma', 'v_gain_sigma', 'w_gain_sigma'):
        for v in (-1e-3, nan, inf):
            out.append({k: v})
    for v in (-1e-3, 1.001, nan):
        out.append({'dropout': v})
    out.append({'stream_id': 1 << 24})
    return out


def _struct(**kw):
    d = dict(range_sigma=0.1, dropout=0.1, v_gain_sigma=0.1, w_gain_sigma=0.1, seed=0, stream_id=0)
    d.update(kw)
    return _lib.NoiseParams(d['range_sigma'], d['dropout'], d['v_gain_sigma'], d['w_gain_sigma'], d['seed'],
                            d['stream_id'])


def _entries(lib, cfg, p, buf, buf2):
    """each entry called with valid buffers; the device entries never reach a launch when an argument is invalid"""
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    return {'scan': lambda: lib.rlca_noise_scan(cfg, p, 0, None, vp(buf), None),
            'action': lambda: lib.rlca_noise_action(cfg, p, 0, vp(buf2), vp(buf2), None),
            'scan_host': lambda: lib.rlca_noise_scan_host(cfg, p, 0, None, vp(buf)),
            'action_host': lambda: lib.rlca_noise_action_host(cfg, p, 0, vp(buf2), vp(buf2))}


@pytest.mark.parametrize('bad', _bad_params(), ids=lambda d: '%s=%r' % next(iter(d.items())))
def test_invalid_params_rejected(built, bad):
    lib = _lib.load()
    cfg = _cfg(4, 2, 8)
    buf, buf2 = _stack(8, 8), np.full((8, 2), 0.5, np.float32)
    keep, keep2 = buf.copy(), buf2.copy()
    for name, call in _entries(lib, C.byref(cfg), C.byref(_struct(**bad)), buf, buf2).items():
        assert call() == 1, name
        assert b'noise' in lib.rlca_last_error()
    assert np.array_equal(_bits(buf), _bits(keep)) and np.array_equal(_bits(buf2), _bits(keep2))


@pytest.mark.parametrize('field,value', [('robots_per_world', 0), ('robots_per_world', 65), ('num_worlds', 0),
                                         ('beams', 0), ('world_offset', -1)])
def test_invalid_config_rejected(built, field, value):
    lib = _lib.load()
    cfg = _cfg(4, 2, 8)
    setattr(cfg, field, value)
    buf, buf2 = _stack(8, 8), np.full((8, 2), 0.5, np.float32)
    for name, call in _entries(lib, C.byref(cfg), C.byref(_struct()), buf, buf2).items():
        assert call() == 1, name


def test_null_pointers_rejected(built):
    lib = _lib.load()
    cfg, p = _cfg(4, 2, 8), _struct()
    buf = np.zeros((8, 2), np.float32)
    vp = buf.ctypes.data_as(C.c_void_p)
    calls = [lib.rlca_noise_scan(None, C.byref(p), 0, None, vp, None),
             lib.rlca_noise_scan(C.byref(cfg), None, 0, None, vp, None),
             lib.rlca_noise_scan(C.byref(cfg), C.byref(p), 0, None, None, None),
             lib.rlca_noise_action(None, C.byref(p), 0, vp, vp, None),
             lib.rlca_noise_action(C.byref(cfg), None, 0, vp, vp, None),
             lib.rlca_noise_action(C.byref(cfg), C.byref(p), 0, None, vp, None),
             lib.rlca_noise_action(C.byref(cfg), C.byref(p), 0, vp, None, None),
             lib.rlca_noise_scan_host(None, C.byref(p), 0, None, vp),
             lib.rlca_noise_scan_host(C.byref(cfg), None, 0, None, vp),
             lib.rlca_noise_scan_host(C.byref(cfg), C.byref(p), 0, None, None),
             lib.rlca_noise_action_host(None, C.byref(p), 0, vp, vp),
             lib.rlca_noise_action_host(C.byref(cfg), None, 0, vp, vp),
             lib.rlca_noise_action_host(C.byref(cfg), C.byref(p), 0, None, vp),
             lib.rlca_noise_action_host(C.byref(cfg), C.byref(p), 0, vp, None)]
    assert calls == [1] * len(calls)


def test_edge_values_accepted(built):
    cfg = _cfg(64, 1, 8)
    st = _stack(64, 8)
    for kw in (dict(dropout=1.0), dict(dropout=0.0), dict(range_sigma=1e30), dict(seed=2 ** 64 - 1)):
        scan_host(cfg, _P(**kw), 2 ** 32 - 1, st, None, stream_id=(1 << 24) - 1)


@pytest.mark.parametrize('kw', [dict(range_sigma=-1.0), dict(dropout=1.5), dict(v_gain_sigma=float('nan')),
                                dict(w_gain_sigma=float('inf')), dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.5)])
def test_noise_params_validated(kw):
    with pytest.raises(ValueError):
        NoiseParams(**kw)


# ------------------------------------------------------------------------------------------------ command lines
def _evaluate_error(argv, capsys):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


POLICY = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')


@pytest.mark.parametrize('argv,msg', [
    (['--baseline', 'orca', '--scan-noise', '0.1'], 'apply to --policy only'),
    (['--baseline', 'nh-orca', '--beam-dropout', '0.1'], 'apply to --policy only'),
    (['--policy', POLICY, '--scan-noise', '-0.1'], 'range_sigma must be finite'),
    (['--policy', POLICY, '--scan-noise', 'nan'], 'range_sigma must be finite'),
    (['--policy', POLICY, '--beam-dropout', '1.5'], 'dropout must be in [0, 1]'),
    (['--policy', POLICY, '--action-noise', '0.1,0.2,0.3'], '--action-noise'),
    (['--policy', POLICY, '--action-noise', 'x'], '--action-noise'),
    (['--policy', POLICY, '--action-noise', '0.1,-1'], 'w_gain_sigma must be finite'),
    (['--policy', POLICY, '--noise-seed', '3'], '--noise-seed applies'),
    (['--policy', POLICY, '--scan-noise', '0.1', '--noise-seed', '-3'], 'noise seed'),
])
def test_evaluate_rejects_bad_noise_flags(built, capsys, argv, msg):
    err = _evaluate_error(['--scenario', 'stage2'] + argv, capsys)
    assert msg in err, err


def test_action_noise_applies_to_baselines(built):
    """--action-noise with a baseline parses; the run itself needs a GPU, so only the argument stage is checked here"""
    import argparse
    from rl_collision_avoidance_b200.noise import add_noise_arguments, noise_from_arguments
    ap = argparse.ArgumentParser()
    add_noise_arguments(ap)
    ap.add_argument('--seed', type=int, default=4)
    assert noise_from_arguments(ap, ap.parse_args([])) is None
    p = noise_from_arguments(ap, ap.parse_args(['--action-noise', '0.1']))
    assert (p.v_gain_sigma, p.w_gain_sigma, p.seed, p.scan_on, p.action_on) == (0.1, 0.1, 4, False, True)
    p = noise_from_arguments(ap, ap.parse_args(['--action-noise', '0.1,0.2', '--scan-noise', '0.05', '--beam-dropout',
                                                '0.3', '--noise-seed', '9']))
    assert (p.range_sigma, p.dropout, p.v_gain_sigma, p.w_gain_sigma, p.seed) == (0.05, 0.3, 0.1, 0.2, 9)


@pytest.mark.parametrize('argv,msg', [
    (['--scan-noise', '-1'], 'range_sigma must be finite'),
    (['--beam-dropout', '2'], 'dropout must be in [0, 1]'),
    (['--action-noise', '0.1,inf'], 'w_gain_sigma must be finite'),
    (['--noise-seed', '1'], '--noise-seed applies'),
])
def test_trainer_rejects_bad_noise_flags(built, capsys, argv, msg):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(argv=argv)
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


def test_kernels_do_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_noise.o')], check=True,
                         capture_output=True, text=True).stdout
    for name in ('rlca_noise_scan_kernelILb0', 'rlca_noise_scan_kernelILb1', 'rlca_noise_action_kernel'):
        m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)' % name, out)
        assert m, out
        assert int(m.group(2)) == 0 and int(m.group(4)) == 0, m.group(0)
        assert int(m.group(1)) <= 40, m.group(0)
