"""The global planner without a GPU (DESIGN.md §9w): the planning graph of the shipped maps and the arenas, the host
twins of the field, waypoint, tracker and reduction entries against an independent restatement (tests/planner_ref.py:
scipy's Dijkstra, a float64 walk), the planner's properties, every refusal (map limit, ABI, evaluate(), the command
line) and the kernels' resources."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import planner_ref as ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.arenas import generate_arenas
from rl_collision_avoidance_b200.planner import MAX_CELLS, NPARTIALS, HostState, PlannerTables, build_plan_tables, \
    check_tables, fields_host, reduce_host, track_host, waypoints_host
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario
from rl_collision_avoidance_b200.worldfile import WorldMap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
F = np.float32


def _cfg(sc, W=1, auto_reset=0, seed=0):
    return fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512, auto_reset=auto_reset, seed=seed)


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _arena_sc(K=8, T=4, seed=0):
    return make_scenario('arena', robots_per_world=K, arenas=T, arena_side=8.0, arena_seed=seed)


def _synthetic(kind, n=40):
    """A 0.2 m map of free cells with walls; the walls of every kind leave gaps a robot passes."""
    c = np.zeros((n, n), np.uint8)
    c[0, :] = c[-1, :] = c[:, 0] = c[:, -1] = 254
    if kind == 'spiral':
        for k, lo in enumerate(range(6, n // 2, 6)):
            hi = n - 1 - lo
            c[lo, lo:hi + 1] = c[hi, lo:hi + 1] = c[lo:hi + 1, lo] = c[lo:hi + 1, hi] = 254
            gap = (lo + 3, lo) if k % 2 == 0 else (hi - 3, hi)
            c[gap[0] - 2:gap[0] + 3, gap[1]] = 0           # a 5-cell door, on alternate sides
    elif kind == 'comb':
        for x in range(8, n - 4, 8):
            if (x // 8) % 2:
                c[1:n - 8, x] = 254
            else:
                c[8:n - 1, x] = 254
    elif kind == 'gaps':
        c[:, n // 2] = 254
        for y in (6, 18, 30):
            c[y - 2:y + 3, n // 2] = 0                      # one-cell-wide traversable gaps through the wall
    return WorldMap(cells=c, resolution=0.2, origin_cx=n // 2, origin_cy=n // 2, init_poses=np.zeros((0, 3)),
                    name='synthetic ' + kind)


def _sc_on(m, R=8):
    """Stage 1's tick constants on map m."""
    return make_scenario('stage1', m, R)


# ---------------------------------------------------------------------------------------------- planning graph
@pytest.mark.parametrize('name', ['stage1', 'stage2'])
def test_tables_of_shipped_maps(name):
    sc = make_scenario(name)
    t = build_plan_tables(sc.map)
    trav = ref.traversable(sc.map.cells, sc.map.resolution)
    assert np.array_equal(t.label >= 0, trav)
    lab, k = ref.components(trav)
    assert np.array_equal(t.label, lab) and t.count == k
    for c in range(k):
        ys, xs = np.nonzero(lab == c)
        assert tuple(t.rects[c]) == (xs.min(), ys.min(), xs.max(), ys.max())
    assert t.max_area <= MAX_CELLS
    check_tables(_cfg(sc), t)


@pytest.mark.parametrize('seed', [0, 1])
def test_each_arena_is_one_planner_component(seed):
    m, at = generate_arenas(16, 8.0, (4, 10), seed=seed)
    t = build_plan_tables(m)
    assert np.array_equal(t.label >= 0, ref.traversable(m.cells, m.resolution))
    for a in range(at.count):
        cx, cy = at.arena_cells(a)
        comp = np.unique(t.label[cy, cx])
        assert len(comp) == 1 and comp[0] >= 0, a
        ys, xs = np.nonzero(t.label == comp[0])
        assert len(xs) == len(cx) and set(zip(xs, ys)) == set(zip(cx, cy)), a


def test_circle_map_is_refused_naming_the_limit():
    with pytest.raises(ValueError, match=r'circle.*over the 58112-cell limit'):
        build_plan_tables(make_scenario('circle').map)


# ---------------------------------------------------------------------------------------------- fields
def _goal_rows(t, m, rng, n, kinds=('trav', 'wall', 'far', 'off')):
    """Goals (n, 4) on traversable cells, non-traversable cells, cells with no traversable cell within 2 and off the
    map's edge, in turn."""
    ocx, ocy, res = m.origin_cx, m.origin_cy, m.resolution
    trav = np.argwhere(t.label >= 0)
    wall = np.argwhere(t.label < 0)
    from scipy import ndimage
    far = np.argwhere(~ndimage.binary_dilation(t.label >= 0, np.ones((5, 5), bool)))
    g = np.zeros((n, 4), np.float32)
    for r in range(n):
        kind = kinds[r % len(kinds)]
        if kind == 'off' or (kind == 'far' and len(far) == 0):
            g[r, :2] = ((m.grid_w - ocx) * res + 0.3, (rng.random() * m.grid_h - ocy) * res)
            continue
        cells = {'trav': trav, 'wall': wall, 'far': far}[kind]
        y, x = cells[rng.integers(len(cells))]
        g[r, :2] = ((x - ocx + rng.random()) * res, (y - ocy + rng.random()) * res)
    return g


def _check_fields(cfg, t, m, st, goal):
    for a in range(len(goal)):
        e = ref.goal_entry(t.label, m.origin_cx, m.origin_cy, F(cfg.ppm), goal[a, 0], goal[a, 1])
        if e is None:
            assert st.entry[a] == -1
            continue
        assert st.entry[a] == e[1] * m.grid_w + e[0]
        rect = tuple(t.rects[t.label[e[1], e[0]]])
        assert tuple(st.rect[a]) == rect
        assert np.array_equal(st.row_field(a), ref.field(t.label, rect, e)), a


@pytest.mark.parametrize('kind', ['stage1', 'arena', 'spiral', 'comb', 'gaps', 'stage2'])
def test_field_twin_equals_dijkstra(built, kind):
    if kind in ('stage1', 'stage2'):
        sc = make_scenario(kind)
    elif kind == 'arena':
        sc = _arena_sc()
    else:
        sc = _sc_on(_synthetic(kind))
    m = sc.map
    t = build_plan_tables(m)
    n = 4 if kind == 'stage2' else 12
    cfg = _cfg(sc, 1)
    cfg.robots_per_world, cfg.num_worlds = n, 1
    goal = _goal_rows(t, m, np.random.default_rng(len(kind)), n)
    st = HostState(cfg, t)
    fields_host(cfg, t, st, goal)
    _check_fields(cfg, t, m, st, goal)
    assert (st.entry >= 0).any() and (st.entry == -1).any()


@pytest.mark.parametrize('kind', ['stage1', 'stage2', 'spiral', 'comb', 'gaps'])
def test_component_graphs_equal_per_field_dijkstra(kind):
    """planner_ref.Graphs, each component's graph built once with numpy shifts, gives ref.field's D for entries in
    every component (a few cells of the big components of the shipped maps, whose per-field graph takes a second)."""
    m = make_scenario(kind).map if kind in ('stage1', 'stage2') else _synthetic(kind)
    t = build_plan_tables(m)
    graphs = ref.Graphs(t.label, t.rects)
    rng = np.random.default_rng(len(kind))
    area = (t.rects[:, 2] - t.rects[:, 0] + 1) * (t.rects[:, 3] - t.rects[:, 1] + 1)
    checked = 0
    for comp in np.argsort(-area):
        ys, xs = np.nonzero(t.label == comp)
        for i in rng.choice(len(xs), size=min(2, len(xs)), replace=False):
            e = (int(xs[i]), int(ys[i]))
            rect, D = graphs.field(e)
            assert rect == tuple(t.rects[comp])
            assert np.array_equal(D, ref.field(t.label, rect, e)), (comp, e)
            checked += 1
        if checked >= 6:
            break
    assert checked >= min(6, 2 * t.count)


def test_only_changed_goal_entries_are_replanned(built):
    sc = make_scenario('stage1')
    t = build_plan_tables(sc.map)
    cfg = _cfg(sc, 1)
    goal = _goal_rows(t, sc.map, np.random.default_rng(1), 24, kinds=('trav',))
    st = HostState(cfg, t)
    fields_host(cfg, t, st, goal)
    assert list(st.replanned()) == list(range(24))
    st.field[3] = 7                                   # a row that is not re-planned keeps whatever it holds
    fields_host(cfg, t, st, goal)
    assert len(st.replanned()) == 0 and (st.field[3] == 7).all()
    goal[5, :2] = goal[9, :2]
    fields_host(cfg, t, st, goal)
    assert list(st.replanned()) == [5]


def _oracle(sc, W, seed, auto_reset):
    from oracle.oracle import OracleWorld, OrcConfig
    ocfg = fill_config(OrcConfig(), sc, num_worlds=W, beams=512, auto_reset=auto_reset, seed=seed)
    return OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)


def _rollout(sc, W, ticks, seed, auto_reset):
    """Yield (meta_in, orc) of an oracle rollout with random actions, after each tick."""
    from helpers import random_actions
    orc = _oracle(sc, W, seed, auto_reset)
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(seed)
    yield None, orc
    for _ in range(ticks):
        meta_in = orc.meta.copy()
        a = random_actions(rng, orc.N)
        a[:, 0] = np.abs(a[:, 0])
        orc.step(a)
        yield meta_in, orc


def test_replans_follow_goal_changes_over_a_stage1_rollout(built):
    sc = make_scenario('stage1')
    t = build_plan_tables(sc.map)
    cfg = _cfg(sc, 2, auto_reset=1, seed=3)
    st = HostState(cfg, t)
    respawns = 0
    prev = None
    for meta_in, orc in _rollout(sc, 2, 60, 3, 1):
        entries = np.array([(lambda e: -1 if e is None else e[1] * sc.map.grid_w + e[0])(
            ref.goal_entry(t.label, sc.map.origin_cx, sc.map.origin_cy, F(cfg.ppm), *orc.goal[a, :2]))
            for a in range(orc.N)], np.int32)
        fields_host(cfg, t, st, orc.goal)
        want = np.arange(orc.N) if prev is None else np.nonzero(entries != prev)[0]
        assert list(st.replanned()) == [a for a in want if entries[a] >= 0]
        if meta_in is not None:
            respawns += int(orc.flags[:, 3].sum())
        prev = entries
    assert respawns > 0


# ---------------------------------------------------------------------------------------------- waypoints
def _waypoint_case(sc, W, seed, auto_reset, ticks):
    t = build_plan_tables(sc.map)
    cfg = _cfg(sc, W, auto_reset=auto_reset, seed=seed)
    st = HostState(cfg, t)
    states = []
    if sc.layout is not None:
        from rl_collision_avoidance_b200.scenarios import arena_layout_host
        orc = _oracle(sc, W, seed, 0)
        orc.reset_world()
        pose, goal, acc, status = arena_layout_host(cfg, sc.layout, orc.pose, orc.goal, orc.acc)
        assert not status.any()
        orc.pose[:], orc.goal[:], orc.acc[:] = pose, goal, acc
        orc.observe()
        from helpers import random_actions
        rng = np.random.default_rng(seed)
        for k in range(ticks):
            states.append((orc.pose.copy(), orc.goal.copy(), orc.gs.copy()))
            orc.step(np.abs(random_actions(rng, orc.N)))
    else:
        for k, (_, orc) in enumerate(_rollout(sc, W, ticks, seed, auto_reset)):
            states.append((orc.pose.copy(), orc.goal.copy(), orc.gs.copy()))
    return cfg, t, st, states


@pytest.mark.parametrize('name', ['stage1', 'stage2', 'arena'])
def test_waypoint_twin_matches_float64_restatement(built, name):
    sc = _arena_sc(8, 4) if name == 'arena' else make_scenario(name)
    W = 4 if name == 'arena' else 1
    cfg, t, st, states = _waypoint_case(sc, W, 5, {'stage1': 1, 'stage2': 2, 'arena': 0}[name], 6)
    m = sc.map
    ppm, res = float(F(cfg.ppm)), float(F(cfg.resolution))
    seen = np.zeros(3, int)
    disagree = 0
    for pose, goal, gs in states:
        fields_host(cfg, t, st, goal)
        out = waypoints_host(cfg, t, st, pose, goal, gs)
        for a in range(len(pose)):
            e = st.entry[a]
            D, rect = (st.row_field(a), tuple(st.rect[a])) if e >= 0 else (None, None)
            s_ref, wp, ch, k = ref.waypoint(t.label, m.origin_cx, m.origin_cy, ppm, res, D, rect, e >= 0, pose[a],
                                            goal[a])
            s = int(st.status[a])
            seen[s] += 1
            if s == 0 or s == 2:
                assert _bits_equal(out[a], gs[a])
            ok = s == s_ref
            if ok and s == 1:
                dx, dy = wp[0] - float(pose[a, 0]), wp[1] - float(pose[a, 1])
                c, sn = math.cos(float(pose[a, 2])), math.sin(float(pose[a, 2]))
                ok = abs(dx * c + dy * sn - out[a, 0]) < 1e-4 and abs(dy * c - dx * sn - out[a, 1]) < 1e-4
                assert _bits_equal(out[a, 2:], gs[a, 2:])
            if not ok:
                # allowed only where a tested segment passes within 1e-5 m of a cell corner
                u, v = float(pose[a, 0]) * ppm, float(pose[a, 1]) * ppm
                near = ref.corner_dist(u, v, float(goal[a, 0]) * ppm, float(goal[a, 1]) * ppm) < 1e-5 * ppm
                for (x, y) in (ch or []):
                    near |= ref.corner_dist(u, v, x - m.origin_cx + 0.5, y - m.origin_cy + 0.5) < 1e-5 * ppm
                assert near, (a, s, s_ref)
                disagree += 1
    assert seen[0] > 0 and (seen[1] > 0 or name != 'stage2')
    assert disagree <= max(1, seen.sum() // 1000), disagree


def test_waypoint_properties(built):
    """Status-0 rows copy gs_in; D strictly decreases along the chain; the waypoint lies on the chain and its segment
    is traversable by the reference's walk; status counts add up."""
    sc = make_scenario('stage2')
    cfg, t, st, states = _waypoint_case(sc, 1, 7, 2, 4)
    m = sc.map
    ppm, res = float(F(cfg.ppm)), float(F(cfg.resolution))
    n1 = 0
    for pose, goal, gs in states:
        fields_host(cfg, t, st, goal)
        out = waypoints_host(cfg, t, st, pose, goal, gs)
        for a in np.nonzero(st.status == 1)[0]:
            D, rect = st.row_field(a), tuple(st.rect[a])
            s_ref, wp, ch, k = ref.waypoint(t.label, m.origin_cx, m.origin_cy, ppm, res, D, rect, True, pose[a], goal[a])
            if s_ref != 1:
                continue
            ds = [ref.field_at(D, rect, x, y) for x, y in ch]
            assert all(d1 < d0 for d0, d1 in zip(ds, ds[1:]))
            x, y = ch[k]
            u, v = float(pose[a, 0]) * ppm, float(pose[a, 1]) * ppm
            assert k == 0 or ref.clear(t.label, m.origin_cx, m.origin_cy, u, v, x - m.origin_cx + 0.5,
                                       y - m.origin_cy + 0.5)
            n1 += 1
        assert _bits_equal(out[st.status != 1], gs[st.status != 1])
    assert n1 > 0
    assert st.status_count.sum() == len(states) * cfg.robots_per_world * cfg.num_worlds


def test_waypoint_keeps_the_speed_of_gs_in(built):
    """A waypoint replaces the local goal only: where gs_in's speed is not the env's goal.zw (a robot parked by a
    re-layout after the tick wrote its gs), every row keeps gs_in's speed."""
    sc = _arena_sc(8, 4)
    cfg, t, st, states = _waypoint_case(sc, 4, 5, 0, 3)
    n1 = 0
    for pose, goal, gs in states:
        gs = gs.copy()
        gs[:, 2:] = goal[:, 2:] + np.float32(0.25)
        fields_host(cfg, t, st, goal)
        out = waypoints_host(cfg, t, st, pose, goal, gs)
        assert _bits_equal(out[:, 2:], gs[:, 2:])
        n1 += int((st.status == 1).sum())
    assert n1 > 0


def test_convex_open_map_sees_every_clear_goal(built):
    n = 48
    c = np.zeros((n, n), np.uint8)
    c[0, :] = c[-1, :] = c[:, 0] = c[:, -1] = 254
    m = WorldMap(cells=c, resolution=0.2, origin_cx=n // 2, origin_cy=n // 2, init_poses=np.zeros((0, 3)), name='box')
    sc = _sc_on(m, 16)
    t = build_plan_tables(m)
    assert t.count == 1
    cfg = _cfg(sc, 4)
    rng = np.random.default_rng(0)
    N = 64
    pose = np.zeros((N, 4), np.float32)
    goal = np.zeros((N, 4), np.float32)
    pose[:, :2] = rng.uniform(-4.5, 4.5, (N, 2))
    pose[:, 2] = rng.uniform(-3, 3, N)
    goal[:, :2] = rng.uniform(-4.5, 4.5, (N, 2))
    gs = rng.standard_normal((N, 4)).astype(np.float32)
    st = HostState(cfg, t)
    fields_host(cfg, t, st, goal)
    out = waypoints_host(cfg, t, st, pose, goal, gs)
    ppm = float(F(cfg.ppm))
    for a in range(N):
        if ref.clear(t.label, m.origin_cx, m.origin_cy, pose[a, 0] * ppm, pose[a, 1] * ppm, goal[a, 0] * ppm,
                     goal[a, 1] * ppm):
            assert st.status[a] == 0 and _bits_equal(out[a], gs[a])


# ---------------------------------------------------------------------------------------------- geodesic tracker
def _track_ref(cfg, t, st, m, meta_in, acc, flags, closed, count, length, records):
    ppm, res = float(F(cfg.ppm)), float(F(cfg.resolution))
    E = records.shape[1]
    for a in range(len(length)):
        start = True
        if flags is not None:
            if closed[a] != meta_in[a, 1] and flags[a, 2] != 0 and count[a] < E:
                records[a, count[a]] = length[a]
            start = flags[a, 3] != 0
        if start:
            e = st.entry[a]
            D, rect = (st.row_field(a), tuple(st.rect[a])) if e >= 0 else (None, None)
            length[a] = ref.geo_length(t.label, m.origin_cx, m.origin_cy, ppm, res, D, rect, e >= 0, acc[a, 2],
                                       acc[a, 3])


def _close_episodes(meta_in, flags, closed, count):
    """The episode tracker's closed / count update of one tick (rlca_eval_track's rule)."""
    for a in range(len(closed)):
        if closed[a] != meta_in[a, 1] and flags[a, 2] != 0:
            count[a] += 1
            closed[a] = meta_in[a, 1]


@pytest.mark.parametrize('name', ['stage1', 'arena'])
def test_tracker_twin_matches_restatement(built, name):
    sc = make_scenario('stage1') if name == 'stage1' else _arena_sc(8, 4)
    W, auto_reset, E = (2, 1, 3) if name == 'stage1' else (4, 0, 1)
    t = build_plan_tables(sc.map)
    cfg = _cfg(sc, W, auto_reset=auto_reset, seed=2)
    st = HostState(cfg, t, episodes=E)
    m = sc.map
    N = cfg.robots_per_world * W
    closed, count = np.full(N, -1, np.int32), np.zeros(N, np.int32)
    length, records = np.full(N, -1.0, np.float32), np.full((N, E), -1.0, np.float32)
    if name == 'arena':
        from helpers import random_actions
        from rl_collision_avoidance_b200.scenarios import arena_layout_host
        orc = _oracle(sc, W, 2, 0)
        orc.reset_world()
        orc.pose[:], orc.goal[:], orc.acc[:], status = arena_layout_host(cfg, sc.layout, orc.pose, orc.goal, orc.acc)
        assert not status.any()
        rng = np.random.default_rng(2)

        def gen():
            yield None, orc
            for _ in range(40):
                mi = orc.meta.copy()
                orc.step(np.abs(random_actions(rng, orc.N)))
                yield mi, orc
        it = gen()
    else:
        it = _rollout(sc, W, 120, 2, 1)
    ends = respawns = 0
    for meta_in, orc in it:
        fields_host(cfg, t, st, orc.goal)
        flags = None if meta_in is None else orc.flags.copy()
        track_host(cfg, t, st, orc.acc, meta_in, flags, closed, count)
        _track_ref(cfg, t, st, m, meta_in, orc.acc, flags, closed, count, length, records)
        assert _bits_equal(st.length, length) and _bits_equal(st.records, records)
        if meta_in is not None:
            ends += int((orc.flags[:, 2] != 0).sum())
            respawns += int(orc.flags[:, 3].sum())
            _close_episodes(meta_in, orc.flags, closed, count)
    assert ends > 0 and (respawns > 0 or name == 'arena')
    assert (records >= 0).any() and (length >= 0).all()


def test_reduce_twin_matches_numpy(built):
    rng = np.random.default_rng(0)
    sc = make_scenario('stage1')
    cfg = _cfg(sc, 3)
    N, E = cfg.robots_per_world * 3, 4
    geo = rng.uniform(0.5, 9.0, (N, E)).astype(np.float32)
    geo[rng.random((N, E)) < 0.1] = -1.0
    erec = np.zeros((N, E, 4), np.float32)
    erec[..., 0] = rng.integers(1, 4, (N, E))
    erec[..., 2] = geo + rng.uniform(-0.6, 3.0, (N, E)).astype(np.float32)
    count = rng.integers(0, E + 2, N).astype(np.int32)
    mask = (rng.random(N) < 0.3).astype(np.uint8)
    r = float(F(cfg.goal_radius))
    for role_mask in (None, mask):
        out = reduce_host(cfg, geo, erec, count, role_mask)
        for w in range(3):
            for row in ((0,) if role_mask is None else (0, 1)):
                s = np.zeros(NPARTIALS)
                for a in range(w * 24, w * 24 + 24):
                    if role_mask is not None and (mask[a] != 0) != row:
                        continue
                    for i in range(min(count[a], E)):
                        L = float(geo[a, i])
                        if not L >= 0:
                            s[4] += 1
                            continue
                        if int(erec[a, i, 0]) != 1:
                            continue
                        x = float(erec[a, i, 2]) - max(L - r, 0.0)
                        s[:4] += (1, L, x, x * x)
                got = out[w] if role_mask is None else out[w, row]
                assert np.allclose(got, s, rtol=1e-12, atol=1e-9)


# ---------------------------------------------------------------------------------------------- refusals
def test_abi_rejects_nulls_and_shapes(built):
    lib = _lib.load()
    sc = make_scenario('stage1')
    t = build_plan_tables(sc.map)
    cfg = _cfg(sc, 1)
    st = HostState(cfg, t)
    goal = np.zeros((24, 4), np.float32)
    es = _lib.EnvState(None, goal.ctypes.data, None, None)
    T, S = t.struct(), st.struct()
    assert lib.rlca_plan_fields_host(C.byref(cfg), C.byref(T), C.byref(S), C.byref(es)) == 0
    assert lib.rlca_plan_fields_host(None, C.byref(T), C.byref(S), C.byref(es)) == 1
    assert lib.rlca_plan_fields_host(C.byref(cfg), None, C.byref(S), C.byref(es)) == 1
    assert lib.rlca_plan_fields_host(C.byref(cfg), C.byref(T), None, C.byref(es)) == 1
    assert lib.rlca_plan_fields_host(C.byref(cfg), C.byref(T), C.byref(S), None) == 1
    assert lib.rlca_plan_fields(C.byref(cfg), C.byref(T), C.byref(S), None, None) == 1
    assert lib.rlca_plan_waypoints_host(C.byref(cfg), C.byref(T), C.byref(S), C.byref(es), None, None) == 1
    assert lib.rlca_plan_waypoints(C.byref(cfg), C.byref(T), C.byref(S), C.byref(es), None, None, None) == 1
    g = np.zeros((24, 4), np.float32)
    assert lib.rlca_plan_waypoints_host(C.byref(cfg), C.byref(T), C.byref(S), C.byref(es), g.ctypes.data,
                                        g.ctypes.data) == 1          # in place: gs_in and gs_out alias
    assert lib.rlca_plan_track_host(C.byref(cfg), C.byref(T), C.byref(S), None, None, None, None, None, 1) == 1
    assert lib.rlca_plan_track(C.byref(cfg), C.byref(T), C.byref(S), None, C.byref(es), None, None, None) == 1
    assert lib.rlca_plan_reduce(C.byref(cfg), C.byref(S), None, 0, 1, None, None) == 1
    assert lib.rlca_plan_reduce_split(C.byref(cfg), C.byref(S), None, None, 0, 1, None, None) == 1
    assert lib.rlca_plan_reduce_host(C.byref(cfg), None, None, None, None, 1, 0, 1, None) == 1
    one = np.zeros(4, np.float32)
    cnt = np.zeros(24, np.int32)
    out = np.zeros(NPARTIALS)
    p = lambda a: a.ctypes.data
    assert lib.rlca_plan_reduce_host(C.byref(cfg), p(one), p(one), p(cnt), None, 0, 0, 1, p(out)) == 1   # episodes
    assert lib.rlca_plan_reduce_host(C.byref(cfg), p(one), p(one), p(cnt), None, 1, 0, 2, p(out)) == 1   # range
    # tables: bad shapes and values
    bad = [PlannerTables(np.full_like(t.label, t.count), t.rects),
           PlannerTables(t.label, np.array(t.rects) + np.array([0, 0, 500, 0], np.int32)),
           PlannerTables(t.label, np.array(t.rects)[:, [2, 1, 0, 3]].copy())]
    for b in bad:
        with pytest.raises(_lib.RlcaError):
            check_tables(cfg, b)
    for field, value in (('max_area', MAX_CELLS + 1), ('max_area', 0), ('num_components', 0), ('label', None)):
        s = t.struct()
        setattr(s, field, value)
        assert lib.rlca_plan_tables_check(C.byref(cfg), C.byref(s)) == 1, field
        assert lib.rlca_plan_fields_host(C.byref(cfg), C.byref(s), C.byref(S), C.byref(es)) == 1, field
    assert lib.rlca_plan_tables_check(None, C.byref(t.struct())) == 1
    cfg2 = _cfg(sc, 1)
    cfg2.robots_per_world = 65
    assert lib.rlca_plan_fields_host(C.byref(cfg2), C.byref(T), C.byref(S), C.byref(es)) == 1


class _Stub:
    def __init__(self, env, **kw):
        self.env = env
        self.__dict__.update(kw)


def test_evaluate_refusals():
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController, OrcaController
    env = object()
    steer = _Stub(env, steer=True)
    with pytest.raises(ValueError, match='the planner belongs to another env'):
        evaluate(env, None, 1, 1, planner=_Stub(object(), steer=True))
    for cls in (OrcaController, NhOrcaController):
        with pytest.raises(ValueError, match='the ORCA baselines read the true goal'):
            evaluate(env, object.__new__(cls), 1, 1, planner=steer)
    with pytest.raises(ValueError, match='the hybrid driver reads the true goal'):
        evaluate(env, None, 1, 1, hybrid=object(), planner=steer)
    with pytest.raises(ValueError, match='localization error needs a planner on the believed pose'):
        evaluate(env, None, 1, 1, localization=_Stub(env), planner=steer)


@pytest.mark.parametrize('argv, message', [
    (['--baseline', 'orca', '--planner'], 'the ORCA baselines read the true goal'),
    (['--baseline', 'nh-orca', '--planner'], 'the ORCA baselines read the true goal'),
    (['--policy', os.path.join(CKPT, 'stage2.pth'), '--hybrid', '--planner'], 'the hybrid driver reads the true goal'),
    (['--policy', os.path.join(CKPT, 'stage2.pth'), '--pose-error', '0.1', '--planner'],
     'localization error needs a planner on the believed pose'),
    (['--policy', os.path.join(CKPT, 'stage2.pth'), '--speed-error', '0.1', '--planner'],
     'localization error needs a planner on the believed pose'),
    (['--policy', os.path.join(CKPT, 'stage2.pth'), '--planner', '--geodesic'], 'give one of --planner and --geodesic'),
    (['--scenario', 'circle', '--baseline', 'nh-orca', '--geodesic'], 'over the 58112-cell limit'),
    (['--scenario', 'circle', '--baseline', 'dwa', '--planner'], 'over the 58112-cell limit'),
])
def test_evaluate_cli_rules(capsys, argv, message):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main((['--scenario', 'stage2'] if '--scenario' not in argv else []) + argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_kernels_do_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_plan.o')], check=True,
                         capture_output=True, text=True).stdout
    for name in ('rlca_plan_list_kernel', 'rlca_plan_field_kernel', 'rlca_plan_waypoints_kernel',
                 'rlca_plan_track_kernel', 'rlca_plan_reduce_kernel'):
        m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % name, out)
        assert m, (name, out)
        assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
        assert int(m.group(1)) <= 64, m.group(0)
