"""Arena layouts without a GPU (DESIGN.md §9v): the generator's map and cell lists, rlca_layout_arena_host and
rlca_layout_arena_respawn_host against a numpy restatement of the rule (tests/arena_ref.py), the properties of the
layouts, every rejected argument (ABI, make_scenario, the command lines), the kernels' resources, and the oracle's tick
on the arena map from host-twin layouts."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest
from scipy import ndimage

import arena_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.arenas import ARENA_DEFAULTS, big_map_reason, generate_arenas, map_shape, \
    placeable_radius
from rl_collision_avoidance_b200.scenarios import ArenaLayout, _footprint_cells, arena_layout_host, \
    arena_relayout_host, arena_tables_struct, fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
_F = np.float32


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ---------------------------------------------------------------------------------------------- generator
def test_generator_is_deterministic_and_seeded():
    m1, t1 = generate_arenas(9, 8.0, (3, 8), seed=5)
    m2, t2 = generate_arenas(9, 8.0, (3, 8), seed=5)
    assert np.array_equal(m1.cells, m2.cells) and (m1.origin_cx, m1.origin_cy) == (m2.origin_cx, m2.origin_cy)
    for a, b in ((t1.cell_off, t2.cell_off), (t1.cells, t2.cells), (t1.rects, t2.rects)):
        assert a.dtype == b.dtype and np.array_equal(a, b)
    m3, t3 = generate_arenas(9, 8.0, (3, 8), seed=6)
    assert not np.array_equal(m1.cells, m3.cells)
    assert t1.cell_off.dtype == np.int32 and t1.cells.dtype == np.int32 and len(t1.cell_off) == 10


def test_map_shape_resolution_and_origin():
    m, t = generate_arenas(64, 10.0, (4, 10), seed=0)
    assert m.resolution == 0.2 and m.cells.shape == (416, 416) and m.grid_w % 16 == 0
    assert (m.origin_cx, m.origin_cy) == (208, 208)
    n = 50
    for a in range(64):
        cx0, cy0, cx1, cy1 = t.rects[a]
        assert (cx1 - cx0 + 1, cy1 - cy0 + 1) == (n, n)
        ring = np.concatenate((m.cells[cy0 - 1, cx0 - 1:cx1 + 2], m.cells[cy1 + 1, cx0 - 1:cx1 + 2],
                               m.cells[cy0 - 1:cy1 + 2, cx0 - 1], m.cells[cy0 - 1:cy1 + 2, cx1 + 1]))
        assert (ring != 0).all(), a
    # the pitch pads a map whose arena grid is not a multiple of 16 cells wide
    m5, _ = generate_arenas(5, 6.0, (0, 2), seed=1)
    assert map_shape(5, 6.0)[5] == 3 * 32 and m5.grid_w == 96 + 0 and m5.origin_cx == 48
    m7, _ = generate_arenas(2, 5.0, (0, 2), seed=1)
    assert m7.grid_w == 64 and map_shape(2, 5.0)[5] == 54 and not m7.cells[:, 54:].any()


@pytest.mark.parametrize('count,side,obstacles,seed', [(64, 10.0, (4, 10), 0), (10, 7.0, (8, 14), 3)])
def test_free_space_never_joins_two_arenas(count, side, obstacles, seed):
    """8-connected flood fill of the free cells: every component lies inside one arena's interior or outside all."""
    m, t = generate_arenas(count, side, obstacles, seed)
    lab, k = ndimage.label(m.cells == 0, structure=np.ones((3, 3), bool))
    owner = np.full(m.cells.shape, -1)
    for a, (cx0, cy0, cx1, cy1) in enumerate(t.rects):
        owner[cy0:cy1 + 1, cx0:cx1 + 1] = a
    for c in range(1, k + 1):
        assert len(np.unique(owner[lab == c])) == 1, c


def _listed_points(m, t, a, rng):
    """World points in arena a's listed cells: the four corners of every cell and jittered interior points."""
    cx, cy = t.arena_cells(a)
    res = m.resolution
    x0, y0 = (cx - m.origin_cx) * res, (cy - m.origin_cy) * res
    pts = [(x0 + dx * res, y0 + dy * res) for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1))]
    for _ in range(3):
        pts.append((x0 + rng.random(len(cx)) * res, y0 + rng.random(len(cx)) * res))
    return np.concatenate([p[0] for p in pts]), np.concatenate([p[1] for p in pts])


@pytest.mark.parametrize('count,side,obstacles,seed', [(16, 10.0, (4, 10), 0), (6, 8.0, (10, 16), 7)])
def test_every_listed_cell_is_placeable(count, side, obstacles, seed):
    """A footprint centred anywhere in a listed cell (corners included), at any heading in [-pi, pi), covers only free
    cells (scenarios._footprint_cells: points every half cell over the rectangle, edges included)."""
    m, t = generate_arenas(count, side, obstacles, seed)
    rng = np.random.default_rng(seed)
    for a in range(count):
        x, y = _listed_points(m, t, a, rng)
        for th in np.linspace(-math.pi, math.pi, 16, endpoint=False):
            rows, cols = _footprint_cells(m, x, y, np.full(len(x), th))
            assert (rows >= 0).all() and (cols >= 0).all() and (rows < m.grid_h).all() and (cols < m.grid_w).all()
            assert not m.cells[rows, cols].any(), (a, th)


def test_placeable_radius_is_the_rule():
    """A cell is listed only when every cell its centre's disc of r_c + res sqrt(2) / 2 meets is free."""
    assert abs(placeable_radius() - (math.hypot(0.22, 0.19) + 0.2 * math.sqrt(2) / 2)) < 1e-6
    m, t = generate_arenas(4, 10.0, (4, 10), 2)
    res, rp = m.resolution, placeable_radius()
    occ = np.argwhere(m.cells != 0)                     # (row, col)
    for a in range(4):
        cx, cy = t.arena_cells(a)
        for i in range(0, len(cx), 7):
            gx = np.maximum(np.abs(occ[:, 1] - cx[i]) - 0.5, 0) * res
            gy = np.maximum(np.abs(occ[:, 0] - cy[i]) - 0.5, 0) * res
            assert (gx * gx + gy * gy > rp * rp).all()


def test_each_list_is_the_largest_4_connected_component():
    m, t = generate_arenas(16, 9.0, (6, 12), 4)
    rp = placeable_radius() / m.resolution
    k = int(math.ceil(rp + 0.5))
    d = np.maximum(np.abs(np.arange(-k, k + 1)) - 0.5, 0)
    struct = d[:, None] ** 2 + d[None, :] ** 2 <= rp * rp
    ok = ~ndimage.binary_dilation(m.cells != 0, structure=struct, border_value=1)
    for a, (cx0, cy0, cx1, cy1) in enumerate(t.rects):
        lab, n = ndimage.label(ok[cy0:cy1 + 1, cx0:cx1 + 1])
        sizes = np.bincount(lab.ravel())[1:]
        cx, cy = t.arena_cells(a)
        listed = np.zeros_like(lab, bool)
        listed[cy - cy0, cx - cx0] = True
        comp = lab[cy - cy0, cx - cx0]
        assert len(np.unique(comp)) == 1 and listed.sum() == (lab == comp[0]).sum() == sizes.max()
        assert list(zip(cy, cx)) == sorted(zip(cy, cx))                  # row-major
        _, nl = ndimage.label(listed)
        assert nl == 1


def test_small_arenas_are_redrawn_or_refused():
    # 64 robots 1.2 m apart do not fit into a 5 m arena: refused after the bounded retry
    with pytest.raises(ValueError, match='cannot hold 64 starts'):
        generate_arenas(2, 5.0, (0, 0), seed=0, robots_per_world=64, separation=1.2)
    m, t = generate_arenas(2, 5.0, (0, 0), seed=0, robots_per_world=8, separation=1.2)
    assert t.count == 2


# ---------------------------------------------------------------------------------------------- the size limit
def test_size_limit_is_the_env_rule():
    """big_map_reason agrees with rlca_env_set_map's rule as test_env_maps restates it from the library's tables."""
    from test_env_maps import host_tables, predict_big
    kr, slots, _ = host_tables(0.2)
    for count, side in ((1, 3.0), (64, 10.0), (400, 10.0), (576, 10.0), (577, 10.0), (700, 10.0), (4, 100.0),
                        (2, 160.0), (3000, 3.0)):
        _, _, _, gw, gh, _ = map_shape(count, side)
        assert (big_map_reason(gw, gh, slots=slots) is not None) == predict_big(0.2, gw, gh, 64, slots), (count, side)
    _, _, _, gw, gh, _ = map_shape(64, 10.0)
    fh = ((gw + 2 + 15) // 16 * 16 - 2) * gh * 256
    assert 40 << 20 < fh < 48 << 20                     # about 44 MB


# ---------------------------------------------------------------------------------------------- sampler
def _setup(K, T, seed, W, pick=0, world_offset=0, max_reject=4096, pre_zero=1, fill=0, side=10.0, obstacles=(4, 10),
           arena_seed=0, D=None, L=None):
    sc = make_scenario('arena', robots_per_world=K, arenas=T, arena_side=side, obstacles=obstacles,
                       arena_seed=arena_seed, separation=D, min_travel=L, pick=pick)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512, seed=seed, world_offset=world_offset,
                      max_reject=max_reject)
    cfg.pre_distance_zero = pre_zero
    rng = np.random.default_rng(fill)
    rows = tuple(rng.standard_normal((K * W, 4)).astype(_F) for _ in range(3))
    return sc, cfg, rows


# (K, T, seed, W, pick, world_offset, pre_distance_zero)
REF_CASES = [(2, 4, 0, 6, 0, 0, 1), (8, 64, 3, 20, 0, 0, 1), (8, 64, 4, 12, 1, 0, 0), (16, 9, 1, 10, 1, 5, 1),
             (32, 4, 2, 4, 0, 3, 0), (24, 16, 7, 5, 1, 100, 1)]


@pytest.mark.parametrize('K,T,seed,W,pick,wo,pre_zero', REF_CASES)
def test_host_equals_numpy_restatement(built, K, T, seed, W, pick, wo, pre_zero):
    sc, cfg, (p, g, a) = _setup(K, T, seed, W, pick, wo, pre_zero=pre_zero)
    got = arena_layout_host(cfg, sc.layout, p, g, a)
    want = arena_ref.layout(cfg, sc.layout, pick, p, g, a)
    for name, x, y in zip(('pose', 'goal', 'acc'), got[:3], want[:3]):
        assert _bits_equal(x, y), name
    assert np.array_equal(got[3], want[3]) and not got[3].any()
    assert _bits_equal(got[1][:, 2:4], g[:, 2:4]) and _bits_equal(got[2][:, 0:2], a[:, 0:2])
    if pick == 0:
        assert np.array_equal(want[4], (wo + np.arange(W)) % T)


def test_restatement_covers_the_multi_round_path(built):
    most = 0
    for K, T, seed, W, pick, wo, pre_zero in REF_CASES:
        sc, cfg, (p, g, a) = _setup(K, T, seed, W, pick, wo, pre_zero=pre_zero)
        most = max(most, int(arena_ref.layout(cfg, sc.layout, pick, p, g, a)[5].max()))
    assert most >= 32, most


def test_failing_world_keeps_its_rows(built):
    """K = 12 in a 5 m arena with 8 tries: status 1 + r for the robot that could not be placed (the restatement's), and
    the world's rows keep their bits."""
    sc, cfg, (p, g, a) = _setup(12, 2, 0, 3, side=5.0, obstacles=(0, 0), D=1.2, L=1.0, max_reject=8)
    got = arena_layout_host(cfg, sc.layout, p, g, a)
    want = arena_ref.layout(cfg, sc.layout, 0, p, g, a)
    assert got[3].all() and np.array_equal(got[3], want[3])
    for x, y in zip(got[:3], (p, g, a)):
        assert _bits_equal(x, y)
    r = int(got[3][0]) - 1
    assert (want[5][0][:r] >= 0).all() and (want[5][0][r] < 0).any()


def test_world_rows_do_not_depend_on_num_worlds_or_sharding(built):
    for pick in (0, 1):
        sc, cfg, rows = _setup(8, 16, 2, 120, pick)
        big = arena_layout_host(cfg, sc.layout, *rows)
        parts = []
        for w0, wc in ((0, 3), (3, 67), (70, 50)):
            c = fill_config(_lib.EnvConfig(), sc, num_worlds=wc, beams=512, seed=2, world_offset=w0)
            parts.append(arena_layout_host(c, sc.layout, *(r[w0 * 8:(w0 + wc) * 8] for r in rows)))
        for i in range(4):
            assert _bits_equal(np.concatenate([q[i] for q in parts]), big[i]), (pick, i)


@pytest.mark.parametrize('pick', [0, 1])
def test_layout_properties(built, pick):
    K, T, W = 8, 64, 256
    sc, cfg, rows = _setup(K, T, 11, W, pick)
    pose, goal, acc, status = arena_layout_host(cfg, sc.layout, *rows)
    assert not status.any()
    lay, t, m = sc.layout, sc.layout.tables, sc.map
    res = m.resolution
    cell = lambda x, o: np.floor(x.astype(np.float64) / res).astype(np.int64) + o
    sx, sy, gx, gy = (v.reshape(W, K).astype(np.float64) for v in (pose[:, 0], pose[:, 1], goal[:, 0], goal[:, 1]))
    used = set()
    for w in range(W):
        # one arena per world: every start and goal in the listed cells of one arena
        owners = set()
        for x, y in ((sx[w], sy[w]), (gx[w], gy[w])):
            c = cell(x, m.origin_cx) | (cell(y, m.origin_cy) << 16)
            for ci in c:
                owner = np.searchsorted(t.cell_off, np.flatnonzero(t.cells == ci)[0], side='right') - 1
                owners.add(int(owner))
        assert len(owners) == 1, w
        used |= owners
        if pick == 0:
            assert owners == {w % T}
        d = np.hypot(sx[w][:, None] - sx[w][None], sy[w][:, None] - sy[w][None]) + np.eye(K) * 1e9
        assert d.min() >= lay.separation - 1e-5
        d = np.hypot(gx[w][:, None] - gx[w][None], gy[w][:, None] - gy[w][None]) + np.eye(K) * 1e9
        assert d.min() >= lay.separation - 1e-5
        assert np.hypot(gx[w] - sx[w], gy[w] - sy[w]).min() >= lay.min_travel - 1e-5
    assert len(used) == T if pick == 0 else len(used) > T // 2
    th = pose[:, 2]
    assert (th > -_F(math.pi)).all() and (th <= _F(math.pi)).all()
    assert np.array_equal(acc[:, 2:4], pose[:, 0:2])


# (K, T, seed, W, pick, pre_distance_zero, max_reject)
RELAYOUT_CASES = [(8, 64, 3, 24, 1, 1, 4096), (8, 9, 4, 12, 0, 0, 4096), (16, 16, 5, 12, 1, 1, 4096),
                  (10, 4, 0, 24, 1, 1, 8)]


def _state(K, W, fill):
    """Rows after a tick: world w latches none, some or all of its robots (w mod 3)."""
    rng = np.random.default_rng(fill)
    pose, goal, acc = (rng.standard_normal((K * W, 4)).astype(_F) for _ in range(3))
    meta = np.zeros((K * W, 4), np.int32)
    meta[:, 0] = rng.integers(1, 500, K * W)
    meta[:, 1] = np.repeat(rng.integers(1, 40, W), K)
    meta[:, 2] = rng.integers(0, 2, K * W)
    flags = rng.integers(0, 4, (K * W, 4)).astype(np.uint8)
    flags[:, 3] = 0
    for w in range(W):
        rows = slice(w * K, (w + 1) * K)
        if w % 3 == 2:
            meta[rows, 3] = 1
        elif w % 3 == 1:
            m = rng.integers(0, 2, K)
            m[0], m[-1] = 1, 0
            meta[rows, 3] = rng.permutation(m)
    return pose, goal, acc, meta, flags


@pytest.mark.parametrize('K,T,seed,W,pick,pre_zero,max_reject', RELAYOUT_CASES)
def test_respawn_host_equals_numpy_restatement(built, K, T, seed, W, pick, pre_zero, max_reject):
    sc, cfg, _ = _setup(K, T, seed, W, pick, max_reject=max_reject, pre_zero=pre_zero)
    rows = _state(K, W, seed)
    got = arena_relayout_host(cfg, sc.layout, *rows)
    want = arena_ref.relayout(cfg, sc.layout, pick, *rows)
    for name, x, y in zip(('pose', 'goal', 'acc', 'meta', 'flags', 'live', 'status'), got, want):
        assert _bits_equal(x, y), name
    relaid = got[4][:, 3].reshape(W, K).all(1)
    assert relaid.any()
    if max_reject == 8:
        assert got[6].any()


def test_training_pick_moves_to_new_arenas(built):
    """pick 1: a world's arena differs between episodes; pick 0 keeps it."""
    sc, cfg, _ = _setup(8, 64, 0, 1, pick=1)
    arenas = {arena_ref.arena_of(0, 0, e, 1, 0, 64) for e in range(40)}
    assert len(arenas) > 20
    assert {arena_ref.arena_of(0, 0, e, 0, 7, 64) for e in range(10)} == {7}


# ---------------------------------------------------------------------------------------------- rejections
def test_abi_rejects_bad_arguments(built):
    lib = _lib.load()
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    sc, cfg, (p, g, a) = _setup(8, 4, 0, 2)
    t = sc.layout.tables
    st = np.zeros(2, np.int32)
    good = _lib.LayoutParams(0.0, 1.2, 5.0)
    tab = arena_tables_struct(t)
    bufs = [vp(p), vp(g), vp(a), vp(st)]
    host = lambda c, prm, tb, pick, *b: lib.rlca_layout_arena_host(c, prm, tb, pick, *b)
    assert host(C.byref(cfg), C.byref(good), C.byref(tab), 0, *bufs) == 0
    assert host(C.byref(cfg), C.byref(good), C.byref(tab), 1, *bufs) == 0
    for i in range(4):
        bad = list(bufs)
        bad[i] = None
        assert host(C.byref(cfg), C.byref(good), C.byref(tab), 0, *bad) == 1, i
    assert host(None, C.byref(good), C.byref(tab), 0, *bufs) == 1
    assert host(C.byref(cfg), None, C.byref(tab), 0, *bufs) == 1
    assert host(C.byref(cfg), C.byref(good), None, 0, *bufs) == 1
    for pick in (-1, 2):
        assert host(C.byref(cfg), C.byref(good), C.byref(tab), pick, *bufs) == 1, pick
    for prm in ((0.0, 1.0, 5.0), (0.0, math.nan, 5.0), (0.0, math.inf, 5.0), (0.0, 1.2, -0.1), (0.0, 1.2, math.nan),
                (0.0, 1.2, math.inf)):
        assert host(C.byref(cfg), C.byref(_lib.LayoutParams(*prm)), C.byref(tab), 0, *bufs) == 1, prm
    # side does not apply: any side, and min_travel beyond side sqrt(2), pass
    for prm in ((-1.0, 1.2, 5.0), (math.nan, 1.2, 5.0), (1.0, 1.2, 9.0)):
        assert host(C.byref(cfg), C.byref(_lib.LayoutParams(*prm)), C.byref(tab), 0, *bufs) == 0, prm
    for K in (1, 65):
        c = fill_config(_lib.EnvConfig(), sc, num_worlds=2, beams=512)
        c.robots_per_world = K
        assert host(C.byref(c), C.byref(good), C.byref(tab), 0, *bufs) == 1, K
    for field, v in (('num_worlds', 0), ('max_reject', 0), ('world_offset', -1)):
        c = fill_config(_lib.EnvConfig(), sc, num_worlds=2, beams=512)
        setattr(c, field, v)
        assert host(C.byref(c), C.byref(good), C.byref(tab), 0, *bufs) == 1, field
    # tables
    off, cells = t.cell_off.copy(), t.cells.copy()
    bad_tables = []
    bad_tables.append(_lib.ArenaTables(0, off.ctypes.data, cells.ctypes.data))             # T < 1
    bad_tables.append(_lib.ArenaTables(4, None, cells.ctypes.data))                         # NULL offsets
    bad_tables.append(_lib.ArenaTables(4, off.ctypes.data, None))                           # NULL cells
    empty = off.copy()
    empty[2] = empty[1]
    bad_tables.append(_lib.ArenaTables(4, empty.ctypes.data, cells.ctypes.data))            # an empty arena
    down = off.copy()
    down[2] = down[1] - 1
    bad_tables.append(_lib.ArenaTables(4, down.ctypes.data, cells.ctypes.data))             # decreasing
    start = off.copy()
    start[0] = 1
    bad_tables.append(_lib.ArenaTables(4, start.ctypes.data, cells.ctypes.data))            # not from 0
    for cell in (cfg.grid_w, cfg.grid_h << 16):                                             # off the map
        c2 = cells.copy()
        c2[5] = cell
        bad_tables.append((_lib.ArenaTables(4, off.ctypes.data, c2.ctypes.data), c2))
    for tb in bad_tables:
        tb = tb[0] if isinstance(tb, tuple) else tb
        assert host(C.byref(cfg), C.byref(good), C.byref(tb), 0, *bufs) == 1
        if tb.num_arenas >= 1 and tb.cell_off and tb.cells:
            assert lib.rlca_arena_tables_check(C.byref(cfg), C.byref(tb)) == 1
    assert lib.rlca_arena_tables_check(C.byref(cfg), C.byref(tab)) == 0
    # the respawn twin: the same, and auto_reset must be 0
    meta, flags, live = np.zeros((16, 4), np.int32), np.zeros((16, 4), np.uint8), np.zeros(16, np.uint8)
    rbufs = [vp(p), vp(g), vp(a), vp(meta), vp(flags), vp(live), vp(st)]
    rhost = lambda c, prm, tb, pick, *b: lib.rlca_layout_arena_respawn_host(c, prm, tb, pick, *b)
    assert rhost(C.byref(cfg), C.byref(good), C.byref(tab), 1, *rbufs) == 0
    for i in range(len(rbufs)):
        bad = list(rbufs)
        bad[i] = None
        assert rhost(C.byref(cfg), C.byref(good), C.byref(tab), 1, *bad) == 1, i
    c = fill_config(_lib.EnvConfig(), sc, num_worlds=2, beams=512, auto_reset=True)
    assert rhost(C.byref(c), C.byref(good), C.byref(tab), 1, *rbufs) == 1
    assert rhost(C.byref(cfg), C.byref(good), C.byref(tab), 2, *rbufs) == 1
    assert rhost(C.byref(cfg), C.byref(good), C.byref(bad_tables[3]), 1, *rbufs) == 1
    # the device entries check their arguments before they launch anything
    state = _lib.EnvState(vp(p), vp(g), vp(a), vp(meta))
    dev = lambda c, prm, tb, pick, s, status: lib.rlca_layout_arena(c, prm, tb, pick, s, status, None)
    assert dev(None, C.byref(good), C.byref(tab), 0, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), None, C.byref(tab), 0, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), None, 0, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), C.byref(bad_tables[0]), 0, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), C.byref(bad_tables[1]), 0, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), C.byref(tab), 2, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), C.byref(tab), 0, None, vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(good), C.byref(tab), 0, C.byref(state), None) == 1
    assert dev(C.byref(cfg), C.byref(_lib.LayoutParams(0.0, 1.0, 5.0)), C.byref(tab), 0, C.byref(state), vp(st)) == 1
    rdev = lambda c, tb, pick, s: lib.rlca_layout_arena_respawn(c, C.byref(good), tb, pick, s, vp(flags), vp(live),
                                                                vp(st), None)
    assert rdev(C.byref(c), C.byref(tab), 1, C.byref(state)) == 1                  # auto_reset 1
    assert rdev(C.byref(cfg), None, 1, C.byref(state)) == 1
    s2 = _lib.EnvState(vp(p), vp(g), vp(a), None)
    assert rdev(C.byref(cfg), C.byref(tab), 1, C.byref(s2)) == 1                  # meta NULL


def test_make_scenario_arena():
    sc = make_scenario('arena')
    assert (sc.name, sc.scenario_id, sc.robots_per_world, sc.timeout, sc.w_threshold, sc.pre_distance_zero) == \
        ('arena', 2, 8, 10000, 0.7, 1)
    lay = sc.layout
    assert isinstance(lay, ArenaLayout)
    assert (lay.count, lay.side, lay.obstacles, lay.seed, lay.pick) == (64, 10.0, (4, 10), 0, 0)
    assert lay.separation == float(np.float32(ARENA_DEFAULTS['separation'])) and lay.min_travel == 5.0
    assert not sc.init_tab.any() and not sc.goal_tab.any() and sc.init_tab.shape == (8, 4)
    assert sc.map.cells.shape == (416, 416)
    sc2 = make_scenario('arena', robots_per_world=4, arenas=9, arena_side=6.0, obstacles=(2, 3), arena_seed=4,
                        separation=1.5, min_travel=2.0, pick=1, timeout=77)
    assert (sc2.robots_per_world, sc2.timeout, sc2.layout.pick, sc2.layout.count, sc2.layout.min_travel) == \
        (4, 77, 1, 9, 2.0)
    assert sc2.map.cells.shape == (96, 96)                  # 3 x 3 arenas of 30 + 2 cells
    assert not np.array_equal(make_scenario('arena', arena_seed=1).map.cells, sc.map.cells)


@pytest.mark.parametrize('kw, message', [
    (dict(robots_per_world=1), 'robots_per_world must be in 2..64'),
    (dict(robots_per_world=65), 'robots_per_world must be in 2..64'),
    (dict(arena_side=math.nan), 'side must be finite and >= 2 m'),
    (dict(arena_side=1.0), 'side must be finite and >= 2 m'),
    (dict(min_travel=-0.5), 'min_travel must be in'),
    (dict(min_travel=14.2), 'min_travel must be in'),
    (dict(separation=1.0), 'separation must be finite and > 1.147 m'),
    (dict(separation=math.inf), 'separation must be finite and >'),
    (dict(pick=2), 'pick must be 0 (world) or 1 (draw)'),
    (dict(timeout=0), 'timeout must be an integer >= 1'),
    (dict(arenas=0), 'count must be an integer >= 1'),
    (dict(obstacles=(5, 2)), 'obstacles must be integers 0 <= lo <= hi'),
    (dict(arenas=700), 'off the small-map path: its first-hit table would take 469 MB > 384 MB'),
    (dict(arenas=2, arena_side=200.0), 'off the small-map path'),
    (dict(arenas=2, arena_side=4.0, robots_per_world=40), 'cannot hold 40 starts'),
])
def test_make_scenario_rejects(kw, message):
    with pytest.raises(ValueError, match=re.escape(message)):
        make_scenario('arena', **kw)


def test_arena_parameters_belong_to_arena():
    for name, kw in (('random', dict(arenas=4)), ('circle', dict(arena_seed=1)), ('stage1', dict(obstacles=(1, 2))),
                     ('random', dict(pick=1)), ('stage2', dict(arena_side=5.0))):
        with pytest.raises(ValueError, match='shape the arena scenario only'):
            make_scenario(name, **kw)
    for kw in (dict(radius=3.0), dict(side=10.0)):
        with pytest.raises(ValueError, match='do not shape the arena scenario'):
            make_scenario('arena', **kw)


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'arena', '--arena-robots', '1'], 'robots_per_world must be in 2..64'),
    (['--scenario', 'arena', '--arena-count', '0'], 'count must be an integer >= 1'),
    (['--scenario', 'arena', '--arena-count', '700'], 'off the small-map path'),
    (['--scenario', 'arena', '--arena-side', '1'], 'side must be finite and >= 2 m'),
    (['--scenario', 'arena', '--arena-obstacles', '3'], '--arena-obstacles must be LO,HI'),
    (['--scenario', 'arena', '--arena-obstacles', '5,1'], 'obstacles must be integers 0 <= lo <= hi'),
    (['--scenario', 'arena', '--arena-separation', '1.0'], 'separation must be finite and >'),
    (['--scenario', 'arena', '--arena-min-travel', '15'], 'min_travel must be in'),
    (['--scenario', 'circle', '--arena-robots', '8'], 'apply to --scenario arena only'),
    (['--scenario', 'random', '--arena-seed', '3'], 'apply to --scenario arena only'),
    (['--scenario', 'arena', '--random-robots', '8'], '--random-robots: not with --scenario arena'),
    (['--scenario', 'arena', '--random-side', '8'], '--random-side: not with --scenario arena'),
])
@pytest.mark.parametrize('who', [['--policy', os.path.join(CKPT, 'stage2.pth')], ['--baseline', 'dwa']])
def test_evaluate_cli_rejects_bad_arena(capsys, argv, message, who):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(argv + who)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'arena', '--arena-timeout', '0'], '--arena-timeout must be >= 1'),
    (['--scenario', 'stage2', '--arena-count', '4'], 'apply to --scenario arena only'),
    (['--mix', 'stage2:2,random:3', '--arena-count', '4'], 'apply to --scenario arena or an arena component of --mix'),
    (['--scenario', 'arena', '--random-timeout', '9'], '--random-timeout: not with --scenario arena'),
    (['--mix', 'stage2:2,arena:2', '--arena-count', '700'], 'off the small-map path'),
    (['--mix', 'stage2:2,maze:2'], "unknown scenario 'maze' (one of stage2, circle, random, arena)"),
])
def test_stage2_cli_rejects_bad_arena(capsys, argv, message):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(stage=2, argv=argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_stage1_cli_rejects_arena(capsys):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(stage=1, argv=['--scenario', 'arena'])
    assert e.value.code == 2
    assert '--scenario arena trains with ppo_stage2.py' in capsys.readouterr().err


def test_kernels_do_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_layout.o')], check=True,
                         capture_output=True, text=True).stdout
    for name in ('rlca_layout_arena_kernel', 'rlca_layout_arena_respawn_kernel'):
        m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % name, out)
        assert m, (name, out)
        assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
        assert int(m.group(1)) <= 64, m.group(0)


# ---------------------------------------------------------------------------------------------- oracle
def _oracle(sc, W, seed):
    from oracle.oracle import OracleWorld, OrcConfig
    ocfg = fill_config(OrcConfig(), sc, num_worlds=W, beams=512, auto_reset=False, seed=seed)
    return OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)


@pytest.mark.parametrize('pick', [0, 1])
def test_no_contact_at_spawn_and_oracle_ticks(built, pick):
    """From host-twin layouts on the arena map, a tick without motion crashes no robot (no footprint meets a static
    cell or another robot), and ticks with random actions run from there."""
    from helpers import random_actions
    K, T, W = 12, 64, 64
    sc, cfg, _ = _setup(K, T, 9, W, pick)
    orc = _oracle(sc, W, 9)
    orc.reset_world()
    pose, goal, acc, status = arena_layout_host(cfg, sc.layout, orc.pose, orc.goal, orc.acc)
    assert not status.any()
    orc.pose[:], orc.goal[:], orc.acc[:] = pose, goal, acc
    orc.observe()
    assert orc.obs.min() > -0.5                            # every robot sees free space at its own position
    orc.step(np.zeros((orc.N, 2), np.float32))
    assert not orc.meta[:, 2].any() and not (orc.flags[:, 2] == 2).any()
    rng = np.random.default_rng(0)
    for _ in range(5):
        orc.step(random_actions(rng, orc.N))
    assert np.isfinite(orc.obs).all()
