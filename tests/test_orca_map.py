"""The map-aware ORCA controllers without a GPU (DESIGN.md §9f): the boundary segments of hand grids and of the shipped
maps, the obstacle lines and velocities of the _map host entries against the float64 reference of
tests/orca_map_ref.py, the all-free grid against the map-blind entries, and bad arguments."""
import numpy as np
import pytest

import nh_orca_ref
import orca_map_ref as ref
import orca_ref
from helpers import ORCA_DT, ORCA_VMAX, orca_cfg, orca_sweep_states
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.orca import (DEFAULTS, MAP_MAX_LINES, NH_DEFAULTS, OBSTACLE_TIME_HORIZON,
                                              ObstacleSet, nh_orca_host, nh_orca_polygon, obstacle_range, orca_host)

TAU_O = OBSTACLE_TIME_HORIZON
R_DD = DEFAULTS['radius']
R_NH = float(np.float32(NH_DEFAULTS['radius']) + np.float32(NH_DEFAULTS['tracking_error']))


def map_cfg(worlds, robots, res=0.2, origin=(0, 0)):
    c = orca_cfg(worlds, robots)
    c.resolution, c.ppm = res, np.float32(1.0) / np.float32(res)
    c.origin_cx, c.origin_cy = origin
    return c


def _grid(h, w, cells):
    g = np.zeros((h, w), np.uint8)
    for j, i in cells:
        g[j, i] = 254
    return g


def _rect(g, j0, j1, i0, i1):
    g[j0:j1, i0:i1] = 254
    return g


def hand_grids():
    out = {'empty': np.zeros((6, 7), np.uint8), 'one cell': _grid(5, 5, [(2, 2)])}
    out['L'] = _rect(_rect(np.zeros((8, 8), np.uint8), 2, 6, 2, 3), 2, 3, 2, 6)
    out['ring'] = _rect(np.zeros((9, 9), np.uint8), 2, 7, 2, 7)
    out['ring'][4, 4] = 0
    out['ring'][3:6, 3:6] = 0
    out['corner pair'] = _grid(6, 6, [(2, 2), (3, 3)])
    out['border'] = _rect(_rect(np.zeros((5, 6), np.uint8), 0, 5, 0, 1), 0, 1, 0, 6)
    out['corridor'] = _rect(_rect(np.zeros((7, 9), np.uint8), 2, 3, 1, 8), 4, 5, 1, 8)   # a one-cell gap at row 3
    out['checker'] = _grid(6, 6, [(1, 1), (2, 2), (1, 3), (3, 1), (3, 3), (2, 4)])
    return out


def shipped():
    from rl_collision_avoidance_b200.scenarios import make_scenario
    return {n: make_scenario(n).map for n in ('stage1', 'stage2', 'circle')}


def _check_geometry(cells, res, origin, max_range=1.35):
    cfg = map_cfg(1, 1, res, origin)
    pts, links, _ = ObstacleSet(cfg, cells, max_range).segments()
    S = len(pts)
    if S == 0:
        assert not np.any(cells)
        return
    prev, nxt, cv = links[:, 0], links[:, 1], links[:, 2]
    assert np.array_equal(prev[nxt], np.arange(S)) and np.array_equal(nxt[prev], np.arange(S))
    # closed: each segment ends where the next starts
    assert np.array_equal(pts[:, 2:4], pts[nxt, 0:2])
    # back to grid corners (exact for these resolutions up to the float rounding of each corner)
    c0 = np.rint(pts[:, 0:2].astype(np.float64) / res + np.array(origin)).astype(np.int64)
    c1 = np.rint(pts[:, 2:4].astype(np.float64) / res + np.array(origin)).astype(np.int64)
    assert np.abs(c0 * res - np.array(origin) * res - pts[:, 0:2]).max() <= 1e-4 * max(1.0, res * max(cells.shape))
    d = c1 - c0
    L = np.abs(d).sum(1)
    assert np.all(L >= 1) and np.all((d[:, 0] == 0) | (d[:, 1] == 0))           # axis-aligned, non-empty
    u = d // L[:, None]
    turn = u[prev, 0] * u[:, 1] - u[prev, 1] * u[:, 0]
    assert np.all(turn != 0)                                                    # no two consecutive collinear
    assert np.array_equal(cv != 0, turn > 0)                                    # convex = a left turn
    # every occupied/free cell edge exactly once, occupied on the left
    unit = []
    for k in range(S):
        for s in range(L[k]):
            a = c0[k] + s * u[k]
            unit.append((tuple(a), tuple(a + u[k])))
    assert len(unit) == len(set(unit))
    assert set(unit) == ref.boundary_edges(cells)
    # signed shoelace area = occupied area
    area = 0.5 * float(np.sum(c0[:, 0] * c1[:, 1] - c1[:, 0] * c0[:, 1]))
    assert area == float(np.count_nonzero(cells))


@pytest.mark.parametrize('name', list(hand_grids()))
def test_hand_grid_boundaries(built, name):
    _check_geometry(hand_grids()[name], 0.2, (3, 2))


def test_corner_touching_cells_share_one_loop(built):
    pts, links, _ = ObstacleSet(map_cfg(1, 1), hand_grids()['corner pair'], 1.35).segments()
    assert len(pts) == 8                                # one loop round both cells, not two squares
    assert int(np.sum(links[:, 2] == 0)) == 2           # the two right turns at the shared corner


@pytest.mark.parametrize('name', ['stage1', 'stage2', 'circle'])
def test_shipped_map_boundaries(built, name):
    m = shipped()[name]
    _check_geometry(m.cells, m.resolution, (m.origin_cx, m.origin_cy))


@pytest.mark.parametrize('name, max_range', [('stage1', 1.35), ('stage2', 1.35), ('circle', 1.35),
                                             ('stage1', 2.35), ('stage2', 2.35), ('circle', 2.35)])
def test_shipped_maps_build_within_the_candidate_capacity(built, name, max_range):
    m = shipped()[name]
    _, _, longest = ObstacleSet(map_cfg(1, 1, m.resolution, (m.origin_cx, m.origin_cy)), m.cells, max_range).segments()
    assert 0 < longest <= 512


def test_too_long_a_list_is_unsupported(built):
    g = np.zeros((200, 200), np.uint8)
    g[::2, ::2] = 254                                   # isolated cells: 4 segments each
    with pytest.raises(_lib.RlcaError, match='RLCA_ORCA_MAP_MAX_CANDIDATES'):
        ObstacleSet(map_cfg(1, 1, 0.05, (100, 100)), g, 1.35)


# ---------------------------------------------------------------------------------------------- agents near walls
def hand_world():
    """A 8 m x 8 m room at 0.2 m: border walls, an L, a ring with a hole, two corner-touching blocks, a 0.8 m corridor
    between two walls; origin at its centre."""
    g = np.zeros((40, 40), np.uint8)
    g[0, :] = g[-1, :] = g[:, 0] = g[:, -1] = 254
    g[5:15, 5:7] = 254
    g[5:7, 5:15] = 254                                  # L
    g[22:30, 22:30] = 254
    g[24:28, 24:28] = 0                                 # ring (hole unreachable)
    g[8:11, 25:28] = 254
    g[11:14, 28:31] = 254                               # blocks touching at a corner
    g[30:32, 4:18] = 254
    g[36:38, 4:18] = 254                                # corridor rows 32-35
    return g, 0.2, (20, 20)


def _sample_states(rng, cells, res, origin, R, W, penetrate=0.1):
    """W worlds of R robots on free cells near walls (some inside walls), random headings, speeds and goals."""
    occ = cells != 0
    H, Wd = cells.shape
    from scipy.ndimage import distance_transform_edt
    dist = distance_transform_edt(~occ) * res
    near = np.argwhere((~occ) & (dist <= 1.2))
    inside = np.argwhere(occ)
    n = R * W
    pick = near[rng.integers(0, len(near), n)]
    wall = rng.random(n) < penetrate
    pick[wall] = inside[rng.integers(0, len(inside), int(wall.sum()))]
    xy = (pick[:, ::-1] - np.array(origin) + rng.random((n, 2))) * res
    pose = np.zeros((n, 4), np.float32)
    goal = np.zeros((n, 4), np.float32)
    meta = np.zeros((n, 4), np.int32)
    pose[:, 0:2], pose[:, 2] = xy, rng.uniform(-np.pi, np.pi, n)
    goal[:, 0:2] = xy + rng.uniform(-6, 6, (n, 2))
    goal[:, 2] = rng.uniform(0, ORCA_VMAX, n)
    meta[:, 2] = rng.random(n) < 0.1
    return pose, goal, meta


def dense_world():
    """Isolated cells at every other cell of a 0.04 m grid inside a 0.5 m disk round the origin: with tau_o = 0.05 s a
    robot near the centre has more obstacle lines than MAP_MAX_LINES, and the bin lists stay under the candidate cap."""
    g = np.zeros((30, 30), np.uint8)
    j, i = np.mgrid[0:30, 0:30]
    disk = np.hypot((i + 0.5 - 15) * 0.04, (j + 0.5 - 15) * 0.04) <= 0.5
    g[::2, ::2] = np.where(disk[::2, ::2], 254, 0)
    return g, 0.04, (15, 15)


DENSE_TAU_O = 0.05


def dense_states(rng, R, W, spread=0.2):
    """W worlds of R robots within `spread` m of the dense world's centre, random headings, speeds and goals."""
    n = R * W
    ang, rad = rng.uniform(-np.pi, np.pi, n), spread * np.sqrt(rng.random(n))
    pose = np.zeros((n, 4), np.float32)
    goal = np.zeros((n, 4), np.float32)
    meta = np.zeros((n, 4), np.int32)
    pose[:, 0], pose[:, 1], pose[:, 2] = rad * np.cos(ang), rad * np.sin(ang), rng.uniform(-np.pi, np.pi, n)
    goal[:, 0:2], goal[:, 2] = rng.uniform(-3, 3, (n, 2)), rng.uniform(0, ORCA_VMAX, n)
    meta[:, 2] = rng.random(n) < 0.1
    return pose, goal, meta


def _worlds():
    g, res, org = hand_world()
    yield 'hand', g, res, org
    for name, m in shipped().items():
        if name != 'circle':
            yield name, m.cells, m.resolution, (m.origin_cx, m.origin_cy)


# status-0 velocities against the float64 LP optimum: as §9d / §9e (an obstacle line crossing another line at a small
# angle magnifies the float32 rounding of both)
STATUS0_TOL = 5e-6


def _check_world(name, cells, res, org, nh, seed, R, W, tau=TAU_O, states=None):
    rng = np.random.default_rng(seed)
    cfg = map_cfg(W, R, res, org)
    r_o = R_NH if nh else R_DD
    obs = ObstacleSet(cfg, cells, obstacle_range(cfg, r_o, tau))
    pts, links, _ = obs.segments()
    S = ref.segment_table(pts, links)
    pose, goal, meta = states(rng, R, W) if states else _sample_states(rng, cells, res, org, R, W)
    p = NH_DEFAULTS if nh else DEFAULTS
    act, vel, st = (nh_orca_host if nh else orca_host)(cfg, pose, goal, meta, **p, obstacles=obs,
                                                       obstacle_time_horizon=tau)
    pos, th, cur = orca_ref.agent_state(pose, goal, meta)
    stats = dict(agents=0, lines=0, dropped=0, status0=0, fallback=0, vo_checked=0, worst_status0=0.0, worst_gap=0.0)
    verts = nh_orca_polygon(cfg) if nh else None
    for a in range(R * W):
        got, dropped = obs.lines(cfg, pose, goal, meta, a, r_o, tau)
        want, wdrop = ref.obstacle_lines(S, pos[a], cur[a], r_o, tau, ORCA_VMAX, MAP_MAX_LINES)
        assert dropped == wdrop == bool(st[a] & 4), (name, a)
        assert len(got) == len(want), (name, a, len(got), len(want))
        for g_, (wp, wd) in zip(got, want):
            assert np.abs(g_[0:2] - wp).max() <= 1e-5 and np.abs(g_[2:4] - wd).max() <= 1e-5, (name, a, g_, wp, wd)
        stats['agents'] += 1
        stats['lines'] += len(got)
        stats['dropped'] += dropped
        Po, no = ref.as_half_planes(want)
        Pa, na = orca_ref.agent_lines(pose, goal, meta, R, a, r_o, p['neighbour_dist'], p['time_horizon'], ORCA_DT)
        Ph, nhp = (nh_orca_ref.polygon_half_planes(verts, th[a]) if nh else (np.zeros((0, 2)), np.zeros((0, 2))))
        v = vel[a].astype(np.float64)
        vpref = orca_ref.preferred(pos[a], goal[a, 0:2], ORCA_VMAX, ORCA_DT)
        hardP, hardn = np.concatenate((Ph, Po)), np.concatenate((nhp, no))
        if st[a] & 1 == 0:
            stats['status0'] += 1
            w = orca_ref.project(np.concatenate((hardP, Pa)), np.concatenate((hardn, na)), ORCA_VMAX, vpref)
            assert w is not None, (name, a)
            err = float(np.abs(v - w).max())
            stats['worst_status0'] = max(stats['worst_status0'], err)
            assert err <= STATUS0_TOL, (name, a, v, w)
            # outside the tau_o velocity obstacle of every segment, by brute force, unless already within r_o
            clear = min(ref.seg_seg_distance(pos[a], pos[a], S['p0'][i], S['p1'][i]) for i in range(len(pts)))
            if clear > r_o + 1e-4 and not st[a] & 4:
                stats['vo_checked'] += 1
                end = pos[a] + tau * v
                for i in range(len(pts)):
                    dd = ref.seg_seg_distance(pos[a], end, S['p0'][i], S['p1'][i])
                    assert dd >= r_o - 1e-5, (name, a, i, dd)
        else:
            stats['fallback'] += 1
            if not st[a] & 2:
                assert len(hardn) == 0 or orca_ref.penetration(hardP, hardn, v).max() <= 1e-6, (name, a)
                if len(na):
                    fstar = _least_penetration(Pa, na, hardP, hardn, ORCA_VMAX)
                    gap = orca_ref.penetration(Pa, na, v).max() - fstar
                    stats['worst_gap'] = max(stats['worst_gap'], abs(gap))
                    assert abs(gap) <= 1e-4, (name, a, gap)
    return stats


def _least_penetration(P, n, Ph, nh, vmax, sides=1440):
    """min over u with the hard half-planes (Ph, nh) and |u| <= vmax (a circumscribed polygon of `sides` edges) of
    the largest penetration into (P, n), by scipy.optimize.linprog."""
    ang = 2 * np.pi * np.arange(sides) / sides
    disk_n = -np.stack((np.cos(ang), np.sin(ang)), 1)
    disk_P = -vmax / np.cos(np.pi / sides) * disk_n
    return nh_orca_ref.least_penetration(P, n, np.concatenate((Ph, disk_P)), np.concatenate((nh, disk_n)))[0]


@pytest.mark.parametrize('nh', [False, True], ids=['orca-dd', 'nh-orca'])
def test_host_entry_against_reference(built, nh):
    totals = {}
    for k, (name, cells, res, org) in enumerate(_worlds()):
        for R, W in ((1, 24), (6, 4), (24, 2)):
            s = _check_world(name, cells, res, org, nh, 100 * k + R, R, W)
            for key, val in s.items():
                totals[key] = max(totals.get(key, 0), val) if key.startswith('worst') else totals.get(key, 0) + val
    assert totals['lines'] > totals['agents']
    assert totals['status0'] > 0 and totals['fallback'] > 0 and totals['vo_checked'] > 0, totals
    print(totals)


@pytest.mark.parametrize('nh', [False, True], ids=['orca-dd', 'nh-orca'])
def test_host_entry_at_the_line_capacity(built, nh):
    """The dense world: agents whose obstacle lines exceed MAP_MAX_LINES keep the nearest 64 (status bit 2), as the
    reference does, and the rest of the checks of test_host_entry_against_reference hold."""
    g, res, org = dense_world()
    totals = {}
    for R, W in ((1, 16), (6, 3)):
        s = _check_world('dense', g, res, org, nh, 7 + R, R, W, tau=DENSE_TAU_O, states=dense_states)
        for key, val in s.items():
            totals[key] = max(totals.get(key, 0), val) if key.startswith('worst') else totals.get(key, 0) + val
    assert totals['dropped'] >= totals['agents'] // 4, totals
    print(totals)


def test_all_free_grid_equals_map_blind(built):
    free = np.zeros((30, 40), np.uint8)
    for nh, p in ((False, DEFAULTS), (True, NH_DEFAULTS)):
        host = nh_orca_host if nh else orca_host
        for (seed, R, W, side), (pose, goal, meta) in orca_sweep_states(range(1, 3), p['neighbour_dist']):
            cfg = map_cfg(W, R, 0.2, (20, 15))
            obs = ObstacleSet(cfg, free, 2.0)
            a = host(cfg, pose, goal, meta, **p)
            b = host(cfg, pose, goal, meta, **p, obstacles=obs)
            for x, y in zip(a, b):
                assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (nh, seed, R)


def test_no_wall_in_range_equals_map_blind(built):
    """A wall farther than the obstacle range changes nothing."""
    g = np.zeros((60, 60), np.uint8)
    g[:, 0] = 254
    cfg = map_cfg(1, 3, 0.2, (0, 30))
    obs = ObstacleSet(cfg, g, 1.35)
    pose = np.zeros((3, 4), np.float32)
    goal = np.zeros((3, 4), np.float32)
    meta = np.zeros((3, 4), np.int32)
    pose[:, 0:2] = [[6, 0], [7, 1], [8, -1]]
    goal[:, 0:2], goal[:, 2] = [[0.5, 0], [6, 0], [7, 5]], 0.8
    a = orca_host(cfg, pose, goal, meta)
    b = orca_host(cfg, pose, goal, meta, obstacles=obs)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


def test_robot_facing_a_wall_stops_short(built):
    """A lone robot driving at a wall: the velocity keeps it r_o / tau_o clear of the wall's grown face."""
    g = np.zeros((20, 20), np.uint8)
    g[:, 15:] = 254                                     # wall face at x = 15 * 0.2 - 2 = 1.0 m
    cfg = map_cfg(1, 1, 0.2, (10, 10))
    obs = ObstacleSet(cfg, g, 1.35)
    pose = np.zeros((1, 4), np.float32)
    goal = np.zeros((1, 4), np.float32)
    meta = np.zeros((1, 4), np.int32)
    goal[0, 0:2], goal[0, 2] = [5.0, 0.0], 1.0
    _, vel, st = orca_host(cfg, pose, goal, meta, obstacles=obs)
    assert st[0] == 0 and abs(vel[0, 0] - (1.0 - R_DD) / TAU_O) <= 1e-6 and abs(vel[0, 1]) <= 1e-6, vel


@pytest.mark.parametrize('bad', [dict(obstacle_time_horizon=0.0), dict(obstacle_time_horizon=float('nan')),
                                 dict(obstacle_time_horizon=float('inf')), dict(obstacle_time_horizon=5.0),
                                 dict(radius=float('inf'))])
def test_bad_arguments_raise(built, bad):
    cfg = map_cfg(1, 1)
    obs = ObstacleSet(cfg, np.zeros((4, 4), np.uint8), 1.35)
    pose, goal, meta = np.zeros((1, 4), np.float32), np.zeros((1, 4), np.float32), np.zeros((1, 4), np.int32)
    for host, p in ((orca_host, DEFAULTS), (nh_orca_host, NH_DEFAULTS)):
        with pytest.raises(_lib.RlcaError):
            host(cfg, pose, goal, meta, **{**p, **bad}, obstacles=obs)


@pytest.mark.parametrize('max_range', [0.0, -1.0, float('nan'), float('inf')])
def test_bad_obstacle_sets_raise(built, max_range):
    with pytest.raises(_lib.RlcaError):
        ObstacleSet(map_cfg(1, 1), np.zeros((4, 4), np.uint8), max_range)


def test_bad_grid_and_config_raise(built):
    cfg = map_cfg(1, 1)
    with pytest.raises(ValueError):
        ObstacleSet(cfg, np.zeros(4, np.uint8), 1.35)
    with pytest.raises(_lib.RlcaError):
        ObstacleSet(cfg, np.zeros((0, 4), np.uint8), 1.35)
    cfg.resolution = 0.0
    with pytest.raises(_lib.RlcaError):
        ObstacleSet(cfg, np.zeros((4, 4), np.uint8), 1.35)


def test_evaluate_py_map_flags(built, capsys):
    import os

    import evaluate as drv
    policy = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'checkpoints', 'stage1_2.pth')
    with pytest.raises(SystemExit):
        drv.main(['--scenario', 'stage1', '--policy', policy, '--orca-map'])
    assert '--orca-map applies to --baseline' in capsys.readouterr().err
    with pytest.raises(SystemExit):
        drv.main(['--scenario', 'stage1', '--baseline', 'orca', '--orca-obstacle-horizon', '2'])
    assert '--orca-obstacle-horizon applies with --orca-map only' in capsys.readouterr().err
