"""Map geometries the environment kernels are tested on (tests/test_env_maps_gpu.py), and their host-side checks.

rlca_env_set_map picks the tick's code path from the map: small maps (first-hit table) or big maps (distance-field
walk), packed inverse records (<= 255 slots) or the plain lists, a 32- or 64-cell footprint window, the outline
slots per edge.  The shipped maps reach two of those combinations; MAP_CASES below are built from seeds so that every
path, the widest small map, maps smaller than the lidar range, off-centre and off-grid origins, open edges and the
template's pitch padding (columns grid_w + 1 .. gw - 1 of the padded template) are compared with the oracle.

CPU: each case's slots, packed flag, kr, oreach and outline slots per edge from the library's own table builders
(rlca_walk_tables_host, rlca_inv_records_host) and the formulas of rlca_env_set_map, and the path they select; and
what the oracle sees from the padding columns of stage 1 (a robot there is outside the floor plan: outside cells are
empty and its rays go on into the map)."""
import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import pytest

from rl_collision_avoidance_b200.worldfile import CELL_STATIC, WorldMap

HALF_LEN, HALF_WID, RANGE_MAX = 0.22, 0.19, 6.0        # scenarios.COMMON


# ------------------------------------------------------------------------------------------------- map builder
def build_map(res, grid_w, grid_h, origin=None, boundary='closed', blobs=0, walls=0, seed=0, keep_free=()):
    """A WorldMap of exactly grid_w x grid_h cells (no pitch alignment).  `origin` (origin_cx, origin_cy) is the cell
    of world (0, 0), default the centre; it may lie outside the grid.  `boundary`: 'closed' (walls on the outer cells),
    'open' (none: robots can drive off the map) or 'gaps' (walls with two openings per side).  `blobs` filled
    rectangles of 0.1-0.8 m and `walls` one-cell-thick straight walls of 1-3 m at seeded places.  `keep_free`: rings
    (r0, r1) in metres round world (0, 0) cleared of blobs and walls (the circle's start footprints)."""
    if boundary not in ('closed', 'open', 'gaps'):
        raise ValueError(boundary)
    rng = np.random.default_rng(seed)
    cells = np.zeros((grid_h, grid_w), np.uint8)
    ox, oy = origin if origin is not None else (grid_w // 2, grid_h // 2)
    inner = np.zeros_like(cells, bool)
    for _ in range(blobs):
        w, h = (max(1, int(rng.uniform(0.1, 0.8) / res)) for _ in range(2))
        x, y = int(rng.integers(0, grid_w)), int(rng.integers(0, grid_h))
        inner[y:y + h, x:x + w] = True
    for _ in range(walls):
        n = max(2, int(rng.uniform(1.0, 3.0) / res))
        x, y = int(rng.integers(0, grid_w)), int(rng.integers(0, grid_h))
        dx, dy = [(1, 0), (0, 1), (1, 1), (1, -1)][int(rng.integers(4))]
        k = np.arange(n)
        xs, ys = x + dx * k, y + dy * k
        ok = (xs >= 0) & (xs < grid_w) & (ys >= 0) & (ys < grid_h)
        inner[ys[ok], xs[ok]] = True
    if keep_free:
        yy, xx = np.mgrid[0:grid_h, 0:grid_w]
        d = np.hypot((xx - ox + 0.5) * res, (yy - oy + 0.5) * res)
        for r0, r1 in keep_free:
            inner &= ~((d >= r0) & (d <= r1))
    cells[inner] = CELL_STATIC
    if boundary in ('closed', 'gaps'):
        cells[0, :] = cells[-1, :] = cells[:, 0] = cells[:, -1] = CELL_STATIC
    if boundary == 'gaps':
        for side in range(4):
            n = grid_w if side < 2 else grid_h
            for _ in range(2):
                a = int(rng.integers(1, n - 1))
                b = min(n - 1, a + max(3, int(rng.uniform(0.6, 1.5) / res)))
                if side == 0:
                    cells[0, a:b] = 0
                elif side == 1:
                    cells[-1, a:b] = 0
                elif side == 2:
                    cells[a:b, 0] = 0
                else:
                    cells[a:b, -1] = 0
    return WorldMap(cells=cells, resolution=res, origin_cx=int(ox), origin_cy=int(oy),
                    init_poses=np.zeros((0, 3)), name=f'test map {grid_w}x{grid_h} @{res}')


# ------------------------------------------------------------------------------------------------- the cases
@dataclass(frozen=True)
class MapCase:
    name: str
    res: float
    grid_w: int
    grid_h: int
    origin: tuple | None       # (origin_cx, origin_cy); None = centred
    boundary: str
    blobs: int
    walls: int
    scenario: str              # 'circle' (K robots on a circle of `radius` round world (0, 0)) or 'stage1'
    K: int
    radius: float
    worlds: int
    ticks: int
    beams: int
    # the path the case is built for (asserted from the library's tables here and by kernel name on the GPU)
    big: bool
    packed: bool
    win: int
    kr: int
    slots: int
    need: tuple                # coverage counters the case must make non-zero (test_env_maps_gpu.py)

    def map(self):
        keep = ((self.radius - 0.5, self.radius + 0.5),) if self.scenario == 'circle' else ()
        return build_map(self.res, self.grid_w, self.grid_h, self.origin, self.boundary, self.blobs, self.walls,
                         seed=self.grid_w * 7 + self.grid_h, keep_free=keep)


ROOM = ('near_static', 'reverted', 'static_hits', 'robot_hits')
MAP_CASES = [
    # 0.25 m: packed records, small map; 57 + 2 = 59 columns in a pitch of 64 (five padding columns)
    MapCase('r025_room_packed', 0.25, 57, 50, None, 'closed', 14, 4, 'circle', 40, 5.0, 3, 120, 512,
            False, True, 32, 25, 188, ROOM),
    # 0.19 m: the first range with 256 slots (no packed records); origin near a corner, walls with gaps, 510 beams
    MapCase('r019_unpacked_corner_b510', 0.19, 70, 64, (24, 22), 'gaps', 10, 4, 'circle', 24, 3.0, 3, 120, 510,
            False, False, 32, 33, 256, ROOM),
    # 0.1 m: grid_w + 2 = 80 (no padding), open edges: robots drive off the map
    MapCase('r010_open_aligned', 0.1, 78, 60, None, 'open', 8, 3, 'circle', 16, 2.4, 3, 150, 512,
            False, False, 32, 61, 484, ROOM + ('outside',)),
    # 0.07 m: range 85.71 cells (not an integer)
    MapCase('r007_fractional_range', 0.07, 150, 130, None, 'closed', 14, 6, 'circle', 32, 3.5, 2, 80, 512,
            False, False, 32, 87, 688, ROOM),
    # 0.05 m, 20 m square: small and unpacked, 64 robots
    MapCase('r005_small_20m', 0.05, 400, 400, None, 'closed', 30, 10, 'circle', 64, 8.0, 2, 60, 512,
            False, False, 32, 121, 972, ROOM),
    # 0.0241 m, 10 m room: kr 250, the largest small-map range; first-hit bytes up to 249 cells
    MapCase('r00241_kr250_small', 0.0241, 415, 415, None, 'closed', 10, 4, 'circle', 24, 3.5, 2, 40, 512,
            False, False, 32, 250, 2056, ROOM + ('far_static',)),
    # 0.024 m, the same room: kr 251, a big map with the 32-cell window
    MapCase('r0024_kr251_big_win32', 0.024, 417, 417, None, 'closed', 10, 4, 'circle', 24, 3.5, 2, 40, 512,
            True, False, 32, 251, 2084, ROOM + ('far_static',)),
    # 0.05 m, 40 m square: big by the first-hit table's size (624 MB), window 32
    MapCase('r005_big_40m', 0.05, 800, 800, None, 'closed', 60, 20, 'circle', 64, 12.0, 2, 50, 512,
            True, False, 32, 121, 972, ROOM),
    # 0.02 m small room: big by kr (301), oreach 16: the 64-cell window
    MapCase('r002_big_win64', 0.02, 250, 200, None, 'closed', 6, 2, 'circle', 12, 1.5, 2, 40, 512,
            True, False, 64, 301, 2508, ROOM),
    # 0.2 m corridors: gw 4096 (the widest small map; outline x in 12 bits up to 4095) and gw 4112 (big by width);
    # world (0, 0) near the right-hand end
    MapCase('r02_corridor_gw4096_small', 0.2, 4094, 30, (4074, 15), 'closed', 40, 6, 'circle', 12, 2.0, 3, 120, 512,
            False, True, 32, 31, 244, ROOM),
    MapCase('r02_corridor_gw4112_big', 0.2, 4095, 30, (4075, 15), 'closed', 40, 6, 'circle', 12, 2.0, 3, 120, 512,
            True, False, 32, 31, 244, ROOM),
    # 4 x 3 m room at 0.1 m: smaller than the lidar range
    MapCase('r01_room_below_range', 0.1, 40, 30, None, 'closed', 2, 1, 'circle', 8, 1.0, 3, 120, 512,
            False, False, 32, 61, 484, ROOM),
    # stage-1 spawns (a disc of 9 m round world (0, 0), no map test) on a map whose origin lies past its right-hand
    # and below its bottom edge: robots spawn and drive on and off the grid
    MapCase('r01_stage1_origin_off_grid', 0.1, 100, 90, (105, -20), 'gaps', 12, 4, 'stage1', 24, 0.0, 3, 150, 512,
            False, False, 32, 61, 484, ('static_hits', 'robot_hits', 'outside', 'reverted')),
]
CASE_IDS = [c.name for c in MAP_CASES]


# ------------------------------------------------------------------------------------------------- set-up formulas
def padded(grid_w, grid_h):
    """rlca_env_set_map's template: one CELL_OOB ring, pitch rounded up to 16."""
    return (grid_w + 2 + 15) // 16 * 16, grid_h + 2


def range_cells(res):
    return float(np.float32(np.float32(1.0 / res)) * np.float32(RANGE_MAX))


def oreach(res):
    """An outline cell is at most this many cells from the robot's centre cell (rlca_env_set_map, in double from the
    float32 config fields)."""
    hl, hw, ppm = float(np.float32(HALF_LEN)), float(np.float32(HALF_WID)), float(np.float32(1.0 / res))
    return math.ceil(math.sqrt(hl * hl + hw * hw) * ppm) + 1


def edge_slots(res):
    """ec = cell_cap / 4R: outline slots per footprint edge."""
    side = 2.0 * max(float(np.float32(HALF_LEN)), float(np.float32(HALF_WID)))
    return 2 * (math.ceil(side * float(np.float32(1.0 / res))) + 1)


def host_tables(res):
    """(kr, slots, packed) as the library's table builders export them for this resolution's range."""
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    rc = C.c_float(range_cells(res))
    kr, ns, ne = C.c_int32(), C.c_int32(), C.c_int32()
    _lib.check(lib.rlca_walk_tables_host(rc, C.byref(kr), C.byref(ns), C.byref(ne), None, None, None, None))
    nrec, novf = C.c_int32(), C.c_int32()
    packed = lib.rlca_inv_records_host(rc, C.byref(nrec), C.byref(novf), None, None) == 0
    return kr.value, ns.value, packed


def predict_big(res, grid_w, grid_h, R, slots):
    """rlca_env_set_map's big-map rule: kr > 250, a first-hit table over 384 MB, gw or gh over 4096, or a small-map
    lidar launch over 100 KB of shared memory (LidarSmem, the outline-cell list, 4 hit[] rows, the warp queues)."""
    gw, gh = padded(grid_w, grid_h)
    kr = math.ceil(range_cells(res)) + 1
    nsp = (slots + 1 + 15) // 16 * 16
    fh = (gw - 2) * (gh - 2) * nsp
    lidar_smem_struct = (6 * 64 * 4 + 64 + 4 + 15) // 16 * 16
    smem = lidar_smem_struct + R * 4 * edge_slots(res) * 4 + 4 * nsp * 4 + 8 * 64 * 4 + 16
    return kr > 250 or fh > (384 << 20) or gw > 4096 or gh > 4096 or smem > 100 * 1024


# (resolution, kr, slots, packed, oreach, window) of the ranges the cases use, and of the shipped maps
TABLE = [(0.25, 25, 188, True, 3, 32), (0.2, 31, 244, True, 3, 32), (0.19, 33, 256, False, 3, 32),
         (0.1, 61, 484, False, 4, 32), (0.07, 87, 688, False, 6, 32), (0.05, 121, 972, False, 7, 32),
         (0.0241, 250, 2056, False, 14, 32), (0.024, 251, 2084, False, 14, 32), (0.02, 301, 2508, False, 16, 64),
         (0.01, 601, 5260, False, 31, 64)]


@pytest.mark.parametrize('res,kr,slots,packed,reach,win', TABLE)
def test_walk_tables_per_resolution(built, res, kr, slots, packed, reach, win):
    assert host_tables(res) == (kr, slots, packed)
    assert oreach(res) == reach and (32 if reach <= 15 else 64) == win
    # ec: every edge's walk fits its outline slots, and the longest walks come close to filling them
    from test_outline_cells import _corners, walk_edge
    rng = np.random.default_rng(int(1 / res))
    longest = 0
    for _ in range(300):
        corn = _corners(rng.uniform(-30, 30), rng.uniform(-30, 30), rng.uniform(-math.pi, math.pi), 1.0 / res)
        for k in range(4):
            longest = max(longest, len(walk_edge(*corn[k], *corn[(k + 1) & 3])))
    assert edge_slots(res) // 2 <= longest <= edge_slots(res)


@pytest.mark.parametrize('case', MAP_CASES, ids=CASE_IDS)
def test_case_takes_the_path_it_names(built, case):
    m = case.map()
    assert (m.grid_w, m.grid_h) == (case.grid_w, case.grid_h)
    kr, slots, packed = host_tables(case.res)
    assert (kr, slots) == (case.kr, case.slots)
    assert predict_big(case.res, case.grid_w, case.grid_h, case.K, slots) == case.big
    # the small-map lidar reads packed records when the range has them; big maps always read the plain lists
    assert (packed and not case.big) == case.packed
    assert (32 if oreach(case.res) <= 15 else 64) == case.win
    if case.scenario == 'circle':                       # the start footprints are on free cells of this map
        from rl_collision_avoidance_b200.scenarios import make_scenario
        sc = make_scenario('circle', map_=m, robots_per_world=case.K, radius=case.radius)
        assert sc.robots_per_world == case.K


def test_cases_cover_every_path():
    paths = {(c.big, c.packed, c.win, c.beams % 32 == 0) for c in MAP_CASES}
    for want in [(False, True, 32, True), (False, False, 32, True), (False, False, 32, False), (True, False, 32, True),
                 (True, False, 64, True)]:
        assert want in paths, want
    pads = {padded(c.grid_w, c.grid_h)[0] - 2 - c.grid_w for c in MAP_CASES}
    assert 0 in pads and max(pads) >= 13                 # pitch with and without padding columns
    assert any(padded(c.grid_w, c.grid_h)[0] == 4096 and not c.big for c in MAP_CASES)
    assert any(padded(c.grid_w, c.grid_h)[0] > 4096 and c.big for c in MAP_CASES)
    assert any(c.grid_w * c.res < RANGE_MAX and c.grid_h * c.res < RANGE_MAX for c in MAP_CASES)
    assert any(c.origin is not None and (c.origin[0] >= c.grid_w or c.origin[1] < 0) for c in MAP_CASES)
    assert {c.boundary for c in MAP_CASES} == {'closed', 'open', 'gaps'}
    assert any(c.scenario == 'stage1' for c in MAP_CASES)


def test_map_builder(built):
    m = build_map(0.1, 78, 60, boundary='open', blobs=5, walls=2, seed=3)
    assert m.cells.shape == (60, 78) and (m.origin_cx, m.origin_cy) == (39, 30)
    assert not m.cells[0].all() and not m.cells[:, 0].all()
    m = build_map(0.1, 40, 30, origin=(-5, 50), boundary='closed', seed=1)
    assert m.cells[0].all() and m.cells[-1].all() and m.cells[:, 0].all() and m.cells[:, -1].all()
    assert (m.origin_cx, m.origin_cy) == (-5, 50)
    g = build_map(0.1, 40, 30, boundary='gaps', seed=1)
    assert not g.cells[0].all() and g.cells[0].any()
    a, b = build_map(0.05, 200, 150, blobs=9, walls=3, seed=4), build_map(0.05, 200, 150, blobs=9, walls=3, seed=4)
    assert np.array_equal(a.cells, b.cells) and a.cells[1:-1, 1:-1].any()


# ------------------------------------------------------------------------------------------------- padding columns
def _solo_oracle(m, poses):
    """The oracle with one robot per world (no other robot in its scan)."""
    from oracle.oracle import OracleWorld, OrcConfig
    from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario
    sc = make_scenario('stage1', map_=m)
    cfg = fill_config(OrcConfig(), sc, num_worlds=len(poses), beams=512)
    cfg.robots_per_world = 1
    return OracleWorld(cfg, m.cells, sc.init_tab[:1], sc.goal_tab[:1])


def test_oracle_sees_the_map_from_the_padding_columns(built):
    """Stage 1: grid_w 112 in a pitch of 128, so padded columns 113 .. 127 are the CELL_OOB ring and padding; x in
    [12.2, 15.0) m are columns 113 .. 126, which a test of the start cell against the pitch (1 <= cx <= gw - 2) would
    take for the floor plan.  A robot there is outside the map; the oracle's rays go on into the map (outside cells are
    empty).  The scans the GPU must give there."""
    from rl_collision_avoidance_b200.scenarios import make_scenario
    m = make_scenario('stage1').map
    res = m.resolution
    gw, _ = padded(m.grid_w, m.grid_h)
    assert (m.grid_w, gw) == (112, 128)
    x0 = (m.grid_w - m.origin_cx) * res               # left edge of the ring column (unpadded column grid_w)
    x1 = (gw - 2 - m.origin_cx) * res                  # right edge of padded column gw - 2
    assert abs(x0 - 12.2) < 1e-9 and abs(x1 - 15.0) < 1e-9
    pose = np.zeros((1, 4), np.float32)
    pose[0, :3] = (13.0, 0.0, np.pi)
    scan = _solo_oracle(m, pose).raycast(pose)[0]
    assert (scan < RANGE_MAX).sum() == 340
    assert abs(float(scan.min()) - 3.0) < 1e-4
    # every padding column: facing the map, the walls are in view
    cols = np.arange(m.grid_w, gw - 1)
    poses = np.zeros((len(cols), 4), np.float32)
    poses[:, 0] = (cols - m.origin_cx + 0.5) * res
    poses[:, 2] = np.pi
    scans = _solo_oracle(m, poses).raycast(poses)
    near = (cols - m.origin_cx + 0.5) * res - x0 < RANGE_MAX - 3.0
    assert np.all((scans < RANGE_MAX).sum(1)[near] > 100)
