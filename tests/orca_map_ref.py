"""Float64 reference of the static-obstacle half-planes of the map-aware ORCA controllers (DESIGN.md §9f), written from
the velocity-obstacle geometry of van den Berg, Guy, Lin, Manocha (2011, §6) and the rules §9f states:

- the occupied/free cell edges of a grid, to check the boundary the library builds;
- per segment, the truncated velocity obstacle as a skeleton scaled by 1 / tau_o (the cut-off segment and two legs,
  legs tangent to the disks of radius r_o round the vertices, by angle), grown by r_o / tau_o; the line is tangent at
  the boundary point nearest to the current velocity, found as the nearest point of the skeleton over all pieces;
- the candidates and their order by the float32 formula §9f fixes, and the covered test, in float64 otherwise.

Nothing here follows the branch structure of the CUDA code.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
COVER_EPS = 1e-5        # a segment is covered when both vertices / tau_o lie at least r_o / tau_o - this beyond a line


def boundary_edges(cells):
    """Every unit cell edge between an occupied and a free cell (cells outside the grid are free), as a set of
    ((x0, y0), (x1, y1)) corner pairs directed with the occupied cell on the left."""
    occ = np.pad(np.asarray(cells) != 0, 1)
    H, W = occ.shape
    out = set()
    for j in range(1, H - 1):
        for i in range(1, W - 1):
            if not occ[j, i]:
                continue
            x, y = i - 1, j - 1
            if not occ[j - 1, i]:
                out.add(((x, y), (x + 1, y)))
            if not occ[j, i + 1]:
                out.add(((x + 1, y), (x + 1, y + 1)))
            if not occ[j + 1, i]:
                out.add(((x + 1, y + 1), (x, y + 1)))
            if not occ[j, i - 1]:
                out.add(((x, y + 1), (x, y)))
    return out


def segment_table(points, links):
    """Per segment: start, end, unit direction, previous / next direction, convex flags (float64)."""
    p0, p1 = points[:, 0:2].astype(np.float64), points[:, 2:4].astype(np.float64)
    d = p1 - p0
    d /= np.hypot(d[:, 0], d[:, 1])[:, None]
    prev, nxt, cv = links[:, 0], links[:, 1], links[:, 2] != 0
    return dict(p0=p0, p1=p1, d=d, pd=d[prev], nd=d[nxt], cv0=cv, cv1=cv[nxt], points=points)


def candidate_keys(points, dirs, pos, range_):
    """(squared distance, index) of the candidates, by §9f's float32 formula, in processing order."""
    px, py = f32(pos[0]), f32(pos[1])
    r1x, r1y = points[:, 0] - px, points[:, 1] - py
    ex, ey = points[:, 2] - points[:, 0], points[:, 3] - points[:, 1]
    t = np.minimum(np.maximum(-(r1x * ex + r1y * ey) / (ex * ex + ey * ey), f32(0)), f32(1))
    qx, qy = r1x + t * ex, r1y + t * ey
    d2 = qx * qx + qy * qy
    free = dirs[:, 0].astype(f32) * -r1y - dirs[:, 1].astype(f32) * -r1x < f32(0)
    ok = np.nonzero((d2 < f32(range_) * f32(range_)) & free)[0]
    order = np.lexsort((ok, d2[ok]))
    return ok[order]


def _rot(u, ang):
    c, s = np.cos(ang), np.sin(ang)
    return np.array([c * u[0] - s * u[1], s * u[0] + c * u[1]])


def _unit(v):
    return v / np.hypot(*v)


def _tangents(c, r):
    """Directions from the origin tangent to the disk (c, r), left and right as seen from the origin."""
    dist = np.hypot(*c)
    a = np.arcsin(r / dist)
    u = c / dist
    return _rot(u, a), _rot(u, -a)


def _ray_nearest(v, o, d):
    t = max(float((v - o) @ d), 0.0)
    return t, o + t * d


def segment_line(pos, vel, S, i, r, tau):
    """The obstacle line of segment i as (point, unit direction), allowed side on the left, or None."""
    a, b, d = S['p0'][i] - pos, S['p1'][i] - pos, S['d'][i]
    e = b - a
    s = -float(a @ e) / float(e @ e)
    q = a + min(max(s, 0.0), 1.0) * e
    if float(q @ q) <= r * r:                                   # the agent overlaps the segment's disk-grown body
        if s < 0:
            return None if not S['cv0'][i] else (np.zeros(2), _unit(np.array([-a[1], a[0]])))
        if s > 1:
            nd = S['nd'][i]
            if not S['cv1'][i] or b[0] * nd[1] - b[1] * nd[0] < 0:   # else the next segment handles it
                return None
            return np.zeros(2), _unit(np.array([-b[1], b[0]]))
        return np.zeros(2), -d
    line_d2 = float((a + s * e) @ (a + s * e))
    lnb, rnb, lcv, rcv = S['pd'][i], S['nd'][i], S['cv0'][i], S['cv1'][i]
    single = False
    if s < 0 and line_d2 <= r * r:                              # seen obliquely: the start vertex alone
        if not S['cv0'][i]:
            return None
        single, c1, c2, rnb, rcv = True, a, a, d, S['cv0'][i]
        ll, rl = _tangents(a, r)
    elif s > 1 and line_d2 <= r * r:                            # the end vertex alone
        if not S['cv1'][i]:
            return None
        single, c1, c2, lnb, lcv = True, b, b, d, S['cv1'][i]
        ll, rl = _tangents(b, r)
    else:
        c1, c2 = a, b
        ll = _tangents(a, r)[0] if S['cv0'][i] else -d         # a leg at a non-convex vertex runs along the segment
        rl = _tangents(b, r)[1] if S['cv1'][i] else d
    lf = bool(lcv) and ll[0] * -lnb[1] - ll[1] * -lnb[0] >= 0   # points into the neighbouring segment: foreign
    rf = bool(rcv) and rl[0] * rnb[1] - rl[1] * rnb[0] <= 0
    if lf:
        ll = -lnb
    if rf:
        rl = rnb
    lc, rc, rt = c1 / tau, c2 / tau, r / tau
    # nearest point of the skeleton (cut-off segment, left ray, right ray) to the velocity
    pieces = []
    if not single:
        cv = rc - lc
        t = min(max(float((vel - lc) @ cv) / float(cv @ cv), 0.0), 1.0)
        pieces.append(('cut', t, lc + t * cv))
    tl, ql = _ray_nearest(vel, lc, ll)
    tr, qr = _ray_nearest(vel, rc, rl)
    pieces += [('left', tl, ql), ('right', tr, qr)]
    dist = [float(np.hypot(*(vel - q))) for _, _, q in pieces]
    kind, t, q = pieces[int(np.argmin(dist))]
    at_left = (kind == 'cut' and t == 0.0) or (kind == 'left' and t == 0.0) or (single and t == 0.0)
    at_right = (kind == 'cut' and t == 1.0) or (kind == 'right' and t == 0.0)
    if at_left or at_right:                                     # a cut-off arc: tangent to the disk there
        c = lc if at_left else rc
        u = _unit(vel - c)
        return c + rt * u, np.array([u[1], -u[0]])
    if kind == 'cut':
        return lc + rt * np.array([d[1], -d[0]]), -d
    if kind == 'left':
        return (None if lf else (lc + rt * np.array([-ll[1], ll[0]]), ll))
    return None if rf else (rc + rt * np.array([rl[1], -rl[0]]), -rl)


def covered(lines, S, i, pos, r, tau):
    for p, dd in lines:
        ok = True
        for v in (S['p0'][i], S['p1'][i]):
            w = (v - pos) / tau - p
            if not w[0] * dd[1] - w[1] * dd[0] - r / tau >= -COVER_EPS:
                ok = False
        if ok:
            return True
    return False


def obstacle_lines(S, pos, vel, r, tau, vmax, cap=None):
    """The obstacle lines of an agent at pos (float64) with current velocity vel, in order; and whether a line found
    no room among `cap`."""
    range_ = f32(f32(tau) * f32(vmax) + f32(r))
    pts = S['points']
    lines = []
    for i in candidate_keys(pts, S['d'], pos, range_):
        if covered(lines, S, i, pos, r, tau):
            continue
        ln = segment_line(pos, vel, S, i, r, tau)
        if ln is None:
            continue
        if cap is not None and len(lines) == cap:
            return lines, True
        lines.append(ln)
    return lines, False


def as_half_planes(lines):
    """(P (k, 2), n (k, 2)) with (v - P) . n >= 0 allowed, as orca_ref takes them."""
    if not lines:
        return np.zeros((0, 2)), np.zeros((0, 2))
    P = np.array([p for p, _ in lines], np.float64)
    D = np.array([d for _, d in lines], np.float64)
    return P, np.stack((-D[:, 1], D[:, 0]), 1)


def seg_seg_distance(a0, a1, b0, b1):
    """Least distance between segments [a0, a1] and [b0, b1] (float64)."""
    def cross(o, p, q):
        return (p[0] - o[0]) * (q[1] - o[1]) - (p[1] - o[1]) * (q[0] - o[0])

    def pt_seg(p, s0, s1):
        e = s1 - s0
        ee = float(e @ e)
        t = 0.0 if ee == 0 else min(max(float((p - s0) @ e) / ee, 0.0), 1.0)
        return float(np.hypot(*(p - s0 - t * e)))
    d1, d2 = cross(a0, a1, b0), cross(a0, a1, b1)
    d3, d4 = cross(b0, b1, a0), cross(b0, b1, a1)
    if d1 * d2 < 0 and d3 * d4 < 0:
        return 0.0
    return min(pt_seg(a0, b0, b1), pt_seg(a1, b0, b1), pt_seg(b0, a0, a1), pt_seg(b1, a0, a1))
