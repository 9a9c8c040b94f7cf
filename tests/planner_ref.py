"""An independent numpy / scipy restatement of the global planner (DESIGN.md §9w) for the CPU tests: traversable
cells, goal entries, the geodesic field by scipy's Dijkstra (one graph per field, or each component's graph built once:
Graphs), the robot entry, the descent chain, a float64 supercover
walk, the waypoint and the geodesic tracker."""
import math

import numpy as np
from scipy import ndimage
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import dijkstra

INF = 0xFFFFFFFF
F = np.float32
NB = ((1, 0), (0, 1), (-1, 0), (0, -1), (1, 1), (-1, 1), (-1, -1), (1, -1))


def traversable(cells, res, half_len=0.22, half_wid=0.19):
    """No non-free cell (cells outside the grid included) whose square comes within r_c + res sqrt(2) / 2 of the cell's
    centre, by an explicit loop over offsets."""
    hl, hw = float(F(half_len)), float(F(half_wid))
    r = (math.sqrt(hl * hl + hw * hw) + float(F(res)) * math.sqrt(2.0) / 2.0) / res
    k = int(math.ceil(r)) + 1
    h, w = cells.shape
    pad = np.ones((h + 2 * k, w + 2 * k), bool)
    pad[k:k + h, k:k + w] = cells != 0
    bad = np.zeros((h, w), bool)
    for di in range(-k, k + 1):
        for dj in range(-k, k + 1):
            gx, gy = max(abs(di) - 0.5, 0.0), max(abs(dj) - 0.5, 0.0)
            if gx * gx + gy * gy <= r * r:
                bad |= pad[k + dj:k + dj + h, k + di:k + di + w]
    return ~bad


def components(trav):
    lab, k = ndimage.label(trav)
    return lab - 1, k


def goal_entry(label, ocx, ocy, ppm, gx, gy):
    """(cx, cy) or None, the float32 rule of rlca_plan.cu restated."""
    h, w = label.shape
    u, v = F(gx) * F(ppm), F(gy) * F(ppm)
    cx, cy = int(np.floor(u)) + ocx, int(np.floor(v)) + ocy
    lab = lambda x, y: label[y, x] if 0 <= x < w and 0 <= y < h else -1
    if lab(cx, cy) >= 0:
        return cx, cy
    best, bd = None, None
    for dy in range(-2, 3):
        for dx in range(-2, 3):
            x, y = cx + dx, cy + dy
            if lab(x, y) < 0:
                continue
            ex, ey = (F(x - ocx) + F(0.5)) - u, (F(y - ocy) + F(0.5)) - v
            d = ex * ex + ey * ey
            if best is None or d < bd:
                best, bd = (x, y), d
    return best


def field(label, rect, entry):
    """(h, w) uint32 D over rect by scipy's Dijkstra on the integer-weighted grid graph of entry's component."""
    x0, y0, x1, y1 = rect
    sub = label[y0:y1 + 1, x0:x1 + 1]
    comp = label[entry[1], entry[0]]
    ins = sub == comp
    h, w = sub.shape
    idx = np.arange(h * w).reshape(h, w)
    rows, cols, wts = [], [], []
    for dx, dy in NB:
        diag = dx != 0 and dy != 0
        for y in range(h):
            for x in range(w):
                nx, ny = x + dx, y + dy
                if not (ins[y, x] and 0 <= nx < w and 0 <= ny < h and ins[ny, nx]):
                    continue
                if diag and not (ins[y, nx] and ins[ny, x]):
                    continue
                rows.append(idx[y, x])
                cols.append(idx[ny, nx])
                wts.append(99 if diag else 70)
    g = coo_matrix((wts, (rows, cols)), shape=(h * w, h * w)).tocsr()
    d = dijkstra(g, indices=idx[entry[1] - y0, entry[0] - x0])
    out = np.full(h * w, INF, np.uint32)
    ok = np.isfinite(d) & ins.ravel()
    out[ok] = d[ok].astype(np.uint32)
    return out.reshape(h, w)


class Graphs:
    """field's graph of every component of `label`, built once per component with numpy shifts over its bounding
    rectangle (rects (K, 4): x0, y0, x1, y1 inclusive), so that each field is one dijkstra call; field(entry) equals
    field(label, rects[comp], entry)."""

    def __init__(self, label, rects):
        self.label = label
        self.rects = [tuple(int(v) for v in r) for r in rects]
        self._graphs = {}

    def graph(self, comp):
        """(csr, (h, w) bool of the component's cells) over the rectangle of component comp"""
        if comp not in self._graphs:
            x0, y0, x1, y1 = self.rects[comp]
            ins = self.label[y0:y1 + 1, x0:x1 + 1] == comp
            h, w = ins.shape
            idx = np.arange(h * w).reshape(h, w)
            rows, cols, wts = [], [], []
            for dx, dy in NB:
                src = (slice(max(0, -dy), h - max(0, dy)), slice(max(0, -dx), w - max(0, dx)))
                dst = (slice(max(0, dy), h + min(0, dy)), slice(max(0, dx), w + min(0, dx)))
                ok = ins[src] & ins[dst]
                diag = dx != 0 and dy != 0
                if diag:
                    ok &= ins[src[0], dst[1]] & ins[dst[0], src[1]]     # both orthogonal neighbours
                rows.append(idx[src][ok])
                cols.append(idx[dst][ok])
                wts.append(np.full(int(ok.sum()), 99 if diag else 70))
            g = coo_matrix((np.concatenate(wts), (np.concatenate(rows), np.concatenate(cols))),
                           shape=(h * w, h * w)).tocsr()
            self._graphs[comp] = (g, ins)
        return self._graphs[comp]

    def field(self, entry):
        """(rect, (h, w) uint32 D over rect) of the goal entry (cx, cy)"""
        comp = int(self.label[entry[1], entry[0]])
        rect = self.rects[comp]
        g, ins = self.graph(comp)
        h, w = ins.shape
        d = dijkstra(g, indices=(entry[1] - rect[1]) * w + entry[0] - rect[0])
        out = np.full(h * w, INF, np.uint32)
        ok = np.isfinite(d) & ins.ravel()
        out[ok] = d[ok].astype(np.uint32)
        return rect, out.reshape(h, w)


def field_at(D, rect, x, y):
    x0, y0, x1, y1 = rect
    if not (x0 <= x <= x1 and y0 <= y <= y1):
        return INF
    return int(D[y - y0, x - x0])


def robot_entry(label, D, rect, comp, cx, cy):
    h, w = label.shape
    if 0 <= cx < w and 0 <= cy < h and label[cy, cx] == comp:
        return cx, cy
    best, bc = INF, None
    for dy in range(-2, 3):
        for dx in range(-2, 3):
            d = field_at(D, rect, cx + dx, cy + dy)
            if d < best:
                best, bc = d, (cx + dx, cy + dy)
    return bc


def chain(D, rect, e, steps=64):
    """The descent chain from entry e: up to `steps` cells, each the allowed neighbour of least D (ties in NB order);
    [e] when e is the goal entry."""
    out, (x, y) = [], e
    while len(out) < steps and field_at(D, rect, x, y) != 0:
        d4 = [field_at(D, rect, x + dx, y + dy) for dx, dy in NB[:4]]
        best, bxy = INF, None
        for k, (dx, dy) in enumerate(NB):
            if k >= 4:
                a, b = (0 if dx > 0 else 2), (1 if dy > 0 else 3)
                if d4[a] == INF or d4[b] == INF:
                    continue
            d = d4[k] if k < 4 else field_at(D, rect, x + dx, y + dy)
            if d < best:
                best, bxy = d, (x + dx, y + dy)
        if bxy is None:
            break
        x, y = bxy
        out.append(bxy)
    return out or [e]


def walk(ax, ay, bx, by):
    """Cells (i, j) (relative to the origin, cell units) the closed segment meets, in float64, column by column."""
    if ax > bx:
        ax, ay, bx, by = bx, by, ax, ay
    i0, i1 = math.floor(ax), math.floor(bx)
    slope = (by - ay) / (bx - ax) if i1 > i0 else 0.0
    cells = []
    for i in range(i0, i1 + 1):
        yl = ay if i == i0 else ay + (i - ax) * slope
        yr = by if i == i1 else ay + (i + 1 - ax) * slope
        for j in range(math.floor(min(yl, yr)), math.floor(max(yl, yr)) + 1):
            cells.append((i, j))
    return cells


def clear(label, ocx, ocy, ax, ay, bx, by):
    h, w = label.shape
    ea, eb = (math.floor(ax), math.floor(ay)), (math.floor(bx), math.floor(by))
    for i, j in walk(ax, ay, bx, by):
        if max(abs(i - ea[0]), abs(j - ea[1])) <= 1 or max(abs(i - eb[0]), abs(j - eb[1])) <= 1:
            continue
        x, y = i + ocx, j + ocy
        if not (0 <= x < w and 0 <= y < h and label[y, x] >= 0):
            return False
    return True


def corner_dist(ax, ay, bx, by):
    """Least distance, in cell units, from the segment to a cell corner (integer point) near it."""
    best = math.inf
    for i, j in walk(ax, ay, bx, by):
        for px, py in ((i, j), (i + 1, j), (i, j + 1), (i + 1, j + 1)):
            dx, dy = bx - ax, by - ay
            L2 = dx * dx + dy * dy
            t = 0.0 if L2 == 0 else min(max(((px - ax) * dx + (py - ay) * dy) / L2, 0.0), 1.0)
            best = min(best, math.hypot(ax + t * dx - px, ay + t * dy - py))
    return best


def waypoint(label, ocx, ocy, ppm, res, D, rect, entry_ok, pose, goal):
    """(status, (wx, wy) or None, chain, the chain index) of one row in float64."""
    u, v = float(pose[0]) * ppm, float(pose[1]) * ppm
    if not entry_ok:
        return 2, None, None, None
    if clear(label, ocx, ocy, u, v, float(goal[0]) * ppm, float(goal[1]) * ppm):
        return 0, None, None, None
    cx, cy = math.floor(u) + ocx, math.floor(v) + ocy
    e = robot_entry(label, D, rect, comp_of(D, rect, label), cx, cy)
    if e is None:
        return 2, None, None, None
    ch = chain(D, rect, e)
    best = 0
    for k, (x, y) in enumerate(ch):
        if clear(label, ocx, ocy, u, v, x - ocx + 0.5, y - ocy + 0.5):
            best = k
    x, y = ch[best]
    return 1, ((x - ocx + 0.5) * res, (y - ocy + 0.5) * res), ch, best


def comp_of(D, rect, label):
    x0, y0, x1, y1 = rect
    ys, xs = np.nonzero(D == 0)
    return label[ys[0] + y0, xs[0] + x0]


def geo_length(label, ocx, ocy, ppm, res, D, rect, has_plan, x, y):
    if not has_plan:
        return -1.0
    cx, cy = int(np.floor(F(x) * F(ppm))) + ocx, int(np.floor(F(y) * F(ppm))) + ocy
    e = robot_entry(label, D, rect, comp_of(D, rect, label), cx, cy)
    if e is None:
        return -1.0
    return float(F(field_at(D, rect, *e) * float(F(res)) / 70.0))
