"""Generated obstacle arenas (DESIGN.md §9v): one map of T walled arenas, each with its own random obstacles, and the
list of cells a robot may be placed in per arena, for the device sampler of rlca_layout_arena.

Map: resolution 0.2 m (stage 1's and stage 2's); arena a sits in column a mod C, row a div C of a C = ceil(sqrt(T))
column grid, a `side` m interior closed by a one-cell wall ring.  An 8-connected walk cannot cross a full row or column
of static cells, so no beam and no robot passes from one arena to another.  World (0, 0) is the map's centre; the
pitch is padded to 16 cells as worldfile.load_world pads it.

Obstacles: n ~ U{lo..hi} per arena, each a rotated rectangle (sides U[0.4, 1.6] m) or a disc (radius U[0.2, 0.8] m),
rasterised FILLED: every cell the closed shape meets, and for a rectangle also the cells of Stage's edge walk
(worldfile._polygon_cells), so the grid holds at least what Stage's edge rasterisation would mark.

Placeable: a cell whose centre has no non-free cell within r_c + res sqrt(2) / 2 (r_c the footprint's circumradius),
so a footprint centred anywhere in the cell, at any heading, covers free cells only.  Of each arena's placeable cells
only the largest 4-connected component is kept, so any start and goal drawn from it are joined by placeable cells.

numpy and scipy only; deterministic in the arguments; runs once, at set-up.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
from scipy import ndimage

from .worldfile import CELL_STATIC, WorldMap, _polygon_cells

RESOLUTION = 0.2
HALF_LEN, HALF_WID = 0.22, 0.19          # scenarios.COMMON's footprint
RANGE_MAX = 6.0
# walk end points of the lidar's range at 0.2 m (rlca_walk_tables_host, 30 cells): rlca_env_set_map's slot count
SLOTS_AT_RES = 244
RECT_SIDES = (0.4, 1.6)
DISC_RADII = (0.2, 0.8)
MAX_REDRAWS = 16
# separation: the random square's 1 m is below the sampler's 2 (r_c + sqrt(2) res) = 1.147 m at 0.2 m
ARENA_DEFAULTS = dict(count=64, side=10.0, obstacles=(4, 10), seed=0, separation=1.2)


@dataclass(frozen=True)
class ArenaTables:
    """The placeable cells of T arenas, as rlca_arena_tables holds them."""
    cell_off: np.ndarray       # (T + 1,) int32: arena a owns cells[cell_off[a]:cell_off[a + 1]]
    cells: np.ndarray          # (cell_off[T],) int32: cx | cy << 16, row-major per arena
    rects: np.ndarray          # (T, 4) int32: interior cells cx0, cy0, cx1, cy1 (inclusive) of each arena

    @property
    def count(self):
        return int(len(self.cell_off) - 1)

    def arena_cells(self, a):
        """(cx, cy) int arrays of arena a's listed cells."""
        c = self.cells[self.cell_off[a]:self.cell_off[a + 1]].astype(np.int64)
        return c & 0xFFFF, c >> 16


def _f32(v):
    return float(np.float32(v))


def placeable_radius(res=RESOLUTION):
    """r_c + res sqrt(2) / 2 in the float32 values the kernels read."""
    hl, hw = _f32(HALF_LEN), _f32(HALF_WID)
    return math.sqrt(hl * hl + hw * hw) + _f32(res) * math.sqrt(2.0) / 2.0


def map_shape(count, side):
    """(cells per arena edge n, grid columns C, rows, grid_w (pitch), grid_h, used width) of `count` arenas."""
    n = int(math.ceil(side / RESOLUTION - 1e-9))
    cols = int(math.ceil(math.sqrt(count)))
    rows = int(math.ceil(count / cols))
    used_w, grid_h = cols * (n + 2), rows * (n + 2)
    return n, cols, rows, (used_w + 15) // 16 * 16, grid_h, used_w


def big_map_reason(grid_w, grid_h, res=RESOLUTION, slots=SLOTS_AT_RES):
    """None when rlca_env_set_map keeps a grid_w x grid_h map at `res` on the small-map path, else which of its limits
    the map passes: kr > 250, a first-hit table over 384 MB ((gw - 2) (gh - 2) nsp bytes) or gw / gh over 4096, for the
    padded template gw = grid_w + 2 rounded up to 16, gh = grid_h + 2."""
    ppm = np.float32(1.0 / res)
    kr = math.ceil(float(ppm * np.float32(RANGE_MAX))) + 1
    gw, gh = (grid_w + 2 + 15) // 16 * 16, grid_h + 2
    nsp = (slots + 1 + 15) // 16 * 16
    fh = (gw - 2) * (gh - 2) * nsp
    if kr > 250:
        return f'the lidar range spans kr = {kr} > 250 cells'
    if fh > 384 << 20:
        return f'its first-hit table would take {fh / 2 ** 20:.0f} MB > 384 MB'
    if gw > 4096 or gh > 4096:
        return f'its padded grid is {gw} x {gh} cells, over 4096'
    return None


def _mark_rect(cells, ocx, ocy, x, y, th, a, b):
    """Fill the rectangle of half sides a, b at (x, y, th) m: the cells it meets (separating axes of the cell square
    and the rectangle) and the cells of Stage's edge walk of its outline."""
    res = RESOLUTION
    c, s = math.cos(th), math.sin(th)
    corners = [(x + c * u - s * v, y + s * u + c * v) for u, v in ((-a, -b), (a, -b), (a, b), (-a, b))]
    xs, ys = [p[0] for p in corners], [p[1] for p in corners]
    i0, i1 = math.floor(min(xs) / res) - 1, math.floor(max(xs) / res) + 1
    j0, j1 = math.floor(min(ys) / res) - 1, math.floor(max(ys) / res) + 1
    ii, jj = np.meshgrid(np.arange(i0, i1 + 1), np.arange(j0, j1 + 1))
    cx, cy = (ii + 0.5) * res - x, (jj + 0.5) * res - y           # cell centres relative to the rectangle's
    h = 0.5 * res
    meet = np.ones(ii.shape, bool)
    for ax, ay, half in ((c, s, a), (-s, c, b)):                   # the rectangle's axes
        proj = cx * ax + cy * ay
        meet &= np.abs(proj) <= half + h * (abs(ax) + abs(ay))
    for ax, ay in ((1.0, 0.0), (0.0, 1.0)):                        # the cell's axes
        proj = cx * ax + cy * ay
        ext = a * abs(c * ax + s * ay) + b * abs(-s * ax + c * ay)
        meet &= np.abs(proj) <= ext + h
    rows, cols = jj[meet] + ocy, ii[meet] + ocx
    edge = np.array(_polygon_cells(corners, 1.0 / res), np.int64).reshape(-1, 2)
    _stamp(cells, np.concatenate((rows, edge[:, 1] + ocy)), np.concatenate((cols, edge[:, 0] + ocx)))


def _mark_disc(cells, ocx, ocy, x, y, r):
    """Fill the disc of radius r at (x, y) m: every cell whose square it meets."""
    res = RESOLUTION
    i0, i1 = math.floor((x - r) / res), math.floor((x + r) / res)
    j0, j1 = math.floor((y - r) / res), math.floor((y + r) / res)
    ii, jj = np.meshgrid(np.arange(i0, i1 + 1), np.arange(j0, j1 + 1))
    dx = np.maximum(np.maximum(ii * res - x, x - (ii + 1) * res), 0.0)
    dy = np.maximum(np.maximum(jj * res - y, y - (jj + 1) * res), 0.0)
    meet = dx * dx + dy * dy <= r * r
    _stamp(cells, jj[meet] + ocy, ii[meet] + ocx)


def _stamp(cells, rows, cols):
    """Mark the cells (rows, cols) that lie on `cells`: an obstacle ends at its arena's wall ring."""
    on = (rows >= 0) & (rows < cells.shape[0]) & (cols >= 0) & (cols < cells.shape[1])
    cells[rows[on], cols[on]] = CELL_STATIC


def _blocked_structure(res=RESOLUTION):
    """The offsets (di, dj) of the cells whose square meets the disc of placeable_radius about a cell's centre."""
    rp = placeable_radius(res) / res
    k = int(math.ceil(rp + 0.5))
    d = np.arange(-k, k + 1)
    gap = np.maximum(np.abs(d) - 0.5, 0.0)
    return gap[:, None] ** 2 + gap[None, :] ** 2 <= rp * rp


def _holds(xs, ys, robots, separation):
    """True when a greedy pass in row-major order finds `robots` cell centres at least `separation` apart."""
    px, py = [], []
    d2 = separation * separation
    for x, y in zip(xs, ys):
        if all((x - qx) ** 2 + (y - qy) ** 2 >= d2 for qx, qy in zip(px, py)):
            px.append(x)
            py.append(y)
            if len(px) >= robots:
                return True
    return False


def generate_arenas(count=64, side=10.0, obstacles=(4, 10), seed=0, robots_per_world=8, separation=1.2):
    """(WorldMap, ArenaTables) of `count` arenas of `side` m with U{lo..hi} obstacles each, drawn from `seed`.  An arena
    whose kept component cannot hold `robots_per_world` starts `separation` m apart is redrawn (up to MAX_REDRAWS
    times, each from its own seed); ValueError after that, for arguments out of range, and for a map that would leave
    rlca_env_set_map's small-map path."""
    T = int(count)
    if T != count or T < 1:
        raise ValueError(f'arena: count must be an integer >= 1, got {count}')
    S = float(side)
    if not (math.isfinite(S) and S >= 2.0):
        raise ValueError(f'arena: side must be finite and >= 2 m, got {side}')
    lo, hi = (int(v) for v in obstacles)
    if not (0 <= lo <= hi) or (lo, hi) != tuple(obstacles):
        raise ValueError(f'arena: obstacles must be integers 0 <= lo <= hi, got {obstacles}')
    n, cols, rows, grid_w, grid_h, used_w = map_shape(T, S)
    why = big_map_reason(grid_w, grid_h)
    if why is not None:
        raise ValueError(f'arena: {T} arenas of {S:g} m make a {grid_w} x {grid_h}-cell map off the small-map path: '
                         f'{why}')
    res = RESOLUTION
    ocx, ocy = used_w // 2, grid_h // 2
    cells = np.zeros((grid_h, grid_w), np.uint8)
    structure = _blocked_structure()
    rects = np.zeros((T, 4), np.int32)
    offs, lists = [0], []
    for a in range(T):
        bx, by = (a % cols) * (n + 2), (a // cols) * (n + 2)          # the arena's wall ring starts here
        cx0, cy0, cx1, cy1 = bx + 1, by + 1, bx + n, by + n            # interior, inclusive
        rects[a] = cx0, cy0, cx1, cy1
        # interior in metres, relative to world (0, 0)
        x0, y0 = (cx0 - ocx) * res, (cy0 - ocy) * res
        for redraw in range(MAX_REDRAWS + 1):
            block = np.zeros((n + 2, n + 2), np.uint8)
            block[0, :] = block[-1, :] = block[:, 0] = block[:, -1] = CELL_STATIC
            rng = np.random.default_rng([int(seed), a, redraw])
            for _ in range(int(rng.integers(lo, hi + 1))):
                x, y = x0 + rng.uniform(0.0, n * res), y0 + rng.uniform(0.0, n * res)
                if rng.random() < 0.5:
                    w2, h2 = rng.uniform(*RECT_SIDES, size=2) / 2
                    _mark_rect(block, ocx - bx, ocy - by, x, y, rng.uniform(0.0, math.pi), w2, h2)
                else:
                    _mark_disc(block, ocx - bx, ocy - by, x, y, rng.uniform(*DISC_RADII))
            block[0, :] = block[-1, :] = block[:, 0] = block[:, -1] = CELL_STATIC
            ok = ~ndimage.binary_dilation(block != 0, structure=structure, border_value=1)
            lab, k = ndimage.label(ok)                       # 4-connected
            if k == 0:
                continue
            sizes = np.bincount(lab.ravel())[1:]
            keep = lab == 1 + int(np.argmax(sizes))          # the largest; ties to the first in row-major order
            jj, ii = np.nonzero(keep)                        # row-major
            if _holds((ii + bx - ocx + 0.5) * res, (jj + by - ocy + 0.5) * res, int(robots_per_world),
                      float(separation)):
                break
        else:
            raise ValueError(f'arena: arena {a} (seed {seed}) cannot hold {robots_per_world} starts {separation:g} m '
                             f'apart after {MAX_REDRAWS} redraws; use fewer robots, a smaller separation or fewer '
                             f'obstacles')
        cells[by:by + n + 2, bx:bx + n + 2] = block
        packed = (ii + bx).astype(np.int64) | ((jj + by).astype(np.int64) << 16)
        lists.append(packed.astype(np.int32))
        offs.append(offs[-1] + len(packed))
    m = WorldMap(cells=cells, resolution=res, origin_cx=int(ocx), origin_cy=int(ocy), init_poses=np.zeros((0, 3)),
                 name=f'arenas T={T} side={S:g} obstacles={lo}..{hi} seed={seed}')
    return m, ArenaTables(np.asarray(offs, np.int32), np.concatenate(lists).astype(np.int32), rects)
