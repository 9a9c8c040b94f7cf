"""Random layouts without a GPU (DESIGN.md §9i): rlca_layout_random_host against a numpy restatement of the rule, the
properties of the layouts it draws, the failure status, every rejected argument (ABI, make_scenario, evaluate.py) and
the register budget of the kernel."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import layout_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.scenarios import Layout, fill_config, make_scenario, random_layout_host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _setup(K, S, D, L, seed, W, world_offset=0, max_reject=4096, pre_zero=1, fill=0):
    sc = make_scenario('random', robots_per_world=K, side=S, separation=D, min_travel=L)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512, seed=seed, world_offset=world_offset,
                      max_reject=max_reject)
    cfg.pre_distance_zero = pre_zero
    rng = np.random.default_rng(fill)
    rows = tuple(rng.standard_normal((K * W, 4)).astype(np.float32) for _ in range(3))
    return sc, cfg, rows


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


# (K, S, D, L, seed, W, pre_distance_zero)
REF_CASES = [(2, 10.0, 1.0, 5.0, 0, 6, 1), (8, 10.0, 1.0, 5.0, 3, 20, 1), (8, 10.0, 1.0, 5.0, 4, 12, 0),
             (64, 20.0, 1.0, 10.0, 1, 3, 1), (64, 12.0, 1.0, 6.0, 2, 3, 0), (32, 8.0, 1.2, 4.0, 7, 4, 1),
             (16, 6.0, 0.7, 0.0, 9, 5, 1)]


@pytest.mark.parametrize('K,S,D,L,seed,W,pre_zero', REF_CASES)
def test_host_equals_numpy_restatement(built, K, S, D, L, seed, W, pre_zero):
    """pose, goal, acc and status of the host twin equal the numpy restatement bit for bit; the fields the layout does
    not write keep their values."""
    sc, cfg, (p, g, a) = _setup(K, S, D, L, seed, W, pre_zero=pre_zero)
    got = random_layout_host(cfg, sc.layout, p, g, a)
    want = layout_ref.layout(cfg, S, D, L, p, g, a)
    for name, x, y in zip(('pose', 'goal', 'acc'), got[:3], want[:3]):
        assert _bits_equal(x, y), name
    assert np.array_equal(got[3], want[3]) and not got[3].any()
    assert _bits_equal(got[1][:, 2:4], g[:, 2:4]) and _bits_equal(got[2][:, 0:2], a[:, 0:2])
    if pre_zero:
        assert not got[0][:, 3].any()
    else:
        d = np.hypot(*(got[1][:, 0:2] - got[0][:, 0:2]).astype(np.float64).T)
        assert np.allclose(got[0][:, 3], d, rtol=1e-6)


def test_numpy_restatement_covers_the_multi_round_path(built):
    """Some robot of REF_CASES needs more than 32 tries, so the comparison covers more than one warp round."""
    most = 0
    for K, S, D, L, seed, W, pre_zero in REF_CASES:
        sc, cfg, (p, g, a) = _setup(K, S, D, L, seed, W, pre_zero=pre_zero)
        most = max(most, int(layout_ref.layout(cfg, S, D, L, p, g, a)[4].max()))
    assert most >= 32, most


def _pairs_min(x, y):
    d = np.hypot(x[:, :, None] - x[:, None, :], y[:, :, None] - y[:, None, :])
    K = x.shape[1]
    return (d + np.eye(K) * 1e9).min(axis=(1, 2))


@pytest.mark.parametrize('K,S,D,L', [(8, 10.0, 1.0, 5.0), (32, 10.0, 1.0, 3.0), (4, 4.0, 0.8, 2.0)])
def test_layout_properties(built, K, S, D, L):
    W = 400
    sc, cfg, (p, g, a) = _setup(K, S, D, L, 11, W)
    pose, goal, acc, status = random_layout_host(cfg, sc.layout, p, g, a)
    assert not status.any()
    sx, sy = pose[:, 0].reshape(W, K).astype(np.float64), pose[:, 1].reshape(W, K).astype(np.float64)
    gx, gy = goal[:, 0].reshape(W, K).astype(np.float64), goal[:, 1].reshape(W, K).astype(np.float64)
    for v in (sx, sy, gx, gy):
        assert np.abs(v).max() <= S / 2
    tol = 1e-5 * S
    assert _pairs_min(sx, sy).min() >= D - tol
    assert _pairs_min(gx, gy).min() >= D - tol
    assert np.hypot(gx - sx, gy - sy).min() >= L - tol
    th = pose[:, 2]
    assert (th > -np.float32(math.pi)).all() and (th <= np.float32(math.pi)).all()
    assert np.array_equal(acc[:, 2:4], pose[:, 0:2])
    rows = pose[:, 0:3].reshape(W, K * 3)
    assert len(np.unique(rows, axis=0)) == W                  # every world has its own layout


def test_seed_repeats_and_changes(built):
    sc, cfg, rows = _setup(8, 10.0, 1.0, 5.0, 5, 16)
    first = random_layout_host(cfg, sc.layout, *rows)
    again = random_layout_host(cfg, sc.layout, *rows)
    for x, y in zip(first, again):
        assert _bits_equal(x, y)
    cfg.seed = 6
    other = random_layout_host(cfg, sc.layout, *rows)
    assert not np.any(np.all(other[0][:, 0:2] == first[0][:, 0:2], axis=1))


def test_world_rows_do_not_depend_on_num_worlds_or_sharding(built):
    """World w's rows are the same with num_worlds 3 and 200, and from handles that hold worlds [0, 70), [70, 200)."""
    K, S, D, L = 8, 10.0, 1.0, 5.0
    sc, cfg, rows = _setup(K, S, D, L, 2, 200)
    big = random_layout_host(cfg, sc.layout, *rows)
    _, cfg3, _ = _setup(K, S, D, L, 2, 3)
    small = random_layout_host(cfg3, sc.layout, *(r[:3 * K] for r in rows))
    for x, y in zip(big[:3], small[:3]):
        assert _bits_equal(x[:3 * K], y)
    parts = []
    for w0, wc in ((0, 70), (70, 130)):
        _, c, _ = _setup(K, S, D, L, 2, wc, world_offset=w0)
        parts.append(random_layout_host(c, sc.layout, *(r[w0 * K:(w0 + wc) * K] for r in rows)))
    for i in range(4):
        assert _bits_equal(np.concatenate([q[i] for q in parts]), big[i])


def test_crowded_layout_fails_and_keeps_rows(built):
    """K = 64 in a 6 m square at 1 m: status 1 + r for the robot that could not be placed (the restatement's), and
    the world's rows keep their bits."""
    sc, cfg, (p, g, a) = _setup(64, 6.0, 1.0, 3.0, 0, 2)
    pose, goal, acc, status = random_layout_host(cfg, sc.layout, p, g, a)
    want = layout_ref.layout(cfg, 6.0, 1.0, 3.0, p, g, a)
    assert status.all() and np.array_equal(status, want[3])
    for x, y in ((pose, p), (goal, g), (acc, a)):
        assert _bits_equal(x, y)
    r = int(status[0]) - 1
    tries = want[4][0]
    assert (tries[:r] >= 0).all() and tries[r, 1] < 0
    # with a budget of 8 tries some worlds of a looser layout are placed and some are not
    sc2, cfg2, rows2 = _setup(16, 8.0, 1.0, 4.0, 0, 8, max_reject=8)
    got2 = random_layout_host(cfg2, sc2.layout, *rows2)
    want2 = layout_ref.layout(cfg2, 8.0, 1.0, 4.0, *rows2)
    assert got2[3].any() and not got2[3].all() and np.array_equal(got2[3], want2[3])
    for x, y in zip(got2[:3], want2[:3]):
        assert _bits_equal(x, y)


# ---------------------------------------------------------------------------------------------- rejections
def _abi_case():
    sc, cfg, (p, g, a) = _setup(8, 10.0, 1.0, 5.0, 0, 2)
    return sc, cfg, p, g, a, np.zeros(2, np.int32)


def test_abi_rejects_bad_arguments(built):
    lib = _lib.load()
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    sc, cfg, p, g, a, st = _abi_case()
    good = _lib.LayoutParams(10.0, 1.0, 5.0)
    host = lambda c, prm, *bufs: lib.rlca_layout_random_host(c, prm, *bufs)
    assert host(C.byref(cfg), C.byref(good), vp(p), vp(g), vp(a), vp(st)) == 0
    bufs = [vp(p), vp(g), vp(a), vp(st)]
    for i in range(4):
        bad = list(bufs)
        bad[i] = None
        assert host(C.byref(cfg), C.byref(good), *bad) == 1, i
    assert host(None, C.byref(good), *bufs) == 1
    assert host(C.byref(cfg), None, *bufs) == 1
    hl, hw, res = (float(np.float32(v)) for v in (cfg.half_len, cfg.half_wid, cfg.resolution))
    bound = 2.0 * (math.sqrt(hl * hl + hw * hw) + math.sqrt(2.0) * res)
    at_bound = np.float32(bound)
    if float(at_bound) > bound:
        at_bound = np.nextafter(at_bound, np.float32(0))
    above = np.nextafter(at_bound, np.float32(np.inf))
    bad_params = [(0.0, 1.0, 0.0), (-1.0, 1.0, 0.0), (math.nan, 1.0, 0.0), (math.inf, 1.0, 0.0),
                  (10.0, 1.0, -0.01), (10.0, 1.0, math.nan), (10.0, 1.0, 14.15), (10.0, 1.0, math.inf),
                  (10.0, float(at_bound), 5.0), (10.0, 0.0, 5.0), (10.0, math.nan, 5.0), (10.0, math.inf, 5.0)]
    for prm in bad_params:
        assert host(C.byref(cfg), C.byref(_lib.LayoutParams(*prm)), *bufs) == 1, prm
    for prm in ((10.0, float(above), 5.0), (10.0, 1.0, 14.142), (10.0, 1.0, 0.0)):
        assert host(C.byref(cfg), C.byref(_lib.LayoutParams(*prm)), *bufs) == 0, prm
    for K in (1, 65, 0):
        c = fill_config(_lib.EnvConfig(), sc, num_worlds=2, beams=512)
        c.robots_per_world = K
        assert host(C.byref(c), C.byref(good), *bufs) == 1, K
    # the device entry checks its arguments before it launches anything
    state = _lib.EnvState(vp(p), vp(g), vp(a), None)
    dev = lambda c, prm, s, status: lib.rlca_layout_random(c, prm, s, status, None)
    assert dev(None, C.byref(good), C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), None, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), None, vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), C.byref(state), None) == 1
    for field in ('pose_dev', 'goal_dev', 'acc_dev'):
        s2 = _lib.EnvState(vp(p), vp(g), vp(a), None)
        setattr(s2, field, None)
        assert dev(C.byref(cfg), C.byref(good), C.byref(s2), vp(st)) == 1, field
    for prm in bad_params:
        assert dev(C.byref(cfg), C.byref(_lib.LayoutParams(*prm)), C.byref(state), vp(st)) == 1, prm


def test_make_scenario_random():
    sc = make_scenario('random')
    assert (sc.name, sc.scenario_id, sc.robots_per_world, sc.timeout, sc.w_threshold, sc.pre_distance_zero) == \
        ('random', 2, 8, 10000, 0.7, 1)
    assert sc.layout == Layout(10.0, 1.0, 5.0)
    assert not sc.init_tab.any() and not sc.goal_tab.any() and sc.init_tab.shape == (8, 4)
    assert np.array_equal(sc.map.cells, make_scenario('circle').map.cells)
    assert make_scenario('random', robots_per_world=64, side=20.0, separation=1.5).layout == Layout(20.0, 1.5, 10.0)
    assert make_scenario('random', side=41.0, min_travel=1.0).layout.side == 41.0
    for name in ('stage1', 'stage2', 'circle'):
        assert make_scenario(name).layout is None


@pytest.mark.parametrize('kw, message', [
    (dict(robots_per_world=1), 'robots_per_world must be in 2..64'),
    (dict(robots_per_world=65), 'robots_per_world must be in 2..64'),
    (dict(side=0.0), 'side must be finite and > 0'),
    (dict(side=-3.0), 'side must be finite and > 0'),
    (dict(side=math.nan), 'side must be finite and > 0'),
    (dict(side=math.inf), 'side must be finite and > 0'),
    (dict(min_travel=-0.5), 'min_travel must be in'),
    (dict(min_travel=14.2), 'min_travel must be in'),
    (dict(min_travel=math.nan), 'min_travel must be in'),
    (dict(separation=0.6), 'separation must be finite and >'),
    (dict(separation=math.nan), 'separation must be finite and >'),
    (dict(separation=math.inf), 'separation must be finite and >'),
    (dict(side=41.5, min_travel=1.0), 'is not on free cells of the map'),
    (dict(side=80.0, min_travel=1.0), 'is not on free cells of the map'),
])
def test_make_scenario_rejects(kw, message):
    with pytest.raises(ValueError, match=re.escape(message)):
        make_scenario('random', **kw)


def test_random_parameters_belong_to_random():
    with pytest.raises(ValueError):
        make_scenario('circle', side=10.0)
    with pytest.raises(ValueError):
        make_scenario('stage1', separation=1.0)
    with pytest.raises(ValueError):
        make_scenario('random', radius=3.0)


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'random', '--random-robots', '1'], 'robots_per_world must be in 2..64'),
    (['--scenario', 'random', '--random-robots', '65'], 'robots_per_world must be in 2..64'),
    (['--scenario', 'random', '--random-side', '0'], 'side must be finite and > 0'),
    (['--scenario', 'random', '--random-side', 'nan'], 'side must be finite and > 0'),
    (['--scenario', 'random', '--random-side', '70'], 'is not on free cells of the map'),
    (['--scenario', 'random', '--random-separation', '0.5'], 'separation must be finite and >'),
    (['--scenario', 'random', '--random-min-travel', '15'], 'min_travel must be in'),
    (['--scenario', 'random', '--random-min-travel', '-1'], 'min_travel must be in'),
    (['--scenario', 'circle', '--random-robots', '8'], 'apply to --scenario random only'),
    (['--scenario', 'stage1', '--random-side', '8'], 'apply to --scenario random only'),
    (['--scenario', 'stage2', '--random-min-travel', '2'], 'apply to --scenario random only'),
    (['--scenario', 'random', '--circle-robots', '8'], '--circle-robots / --circle-radius apply to'),
    (['--scenario', 'random', '--random-robots', '4', '--non-cooperative', '5'], '--non-cooperative must be in 1..4'),
])
@pytest.mark.parametrize('who', [['--policy', os.path.join(CKPT, 'stage2.pth')], ['--baseline', 'orca']])
def test_evaluate_cli_rejects_bad_random(capsys, argv, message, who):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(argv + who)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_default_max_ticks():
    import evaluate
    assert evaluate.random_max_ticks(10.0) == 3 * 142
    assert evaluate.random_max_ticks(20.0) == 3 * 283


def test_kernel_does_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_layout.o')], check=True,
                         capture_output=True, text=True).stdout
    m = re.search(r'Function \w*rlca_layout_random_kernel\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', out)
    assert m, out
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
    assert int(m.group(1)) <= 64, m.group(0)
