"""Float64 reference of the ORCA-DD controller (DESIGN.md §9d), written from van den Berg, Guy, Lin, Manocha,
"Reciprocal n-body collision avoidance" (2011), §4-5, by plain geometry:

- the ORCA half-plane of a pair comes from the point of the velocity obstacle's boundary nearest to the relative
  velocity, found among all boundary pieces (cut-off arc, both leg rays; the one-step disk when the pair overlaps);
- the LP optimum is found by enumerating every point where the optimum of a projection onto a convex set, or of a
  least-maximum of linear functions on a disk, can lie, and keeping the best feasible one.

Nothing here follows the structure of the CUDA code (incremental LPs); only the definitions are shared.
"""
from __future__ import annotations

from functools import lru_cache
from itertools import combinations

import numpy as np

FEAS_TOL = 1e-9


def agent_state(pose, goal, meta):
    """Positions (N, 2), headings (N) and current velocities (N, 2) in float64."""
    p = pose[:, 0:2].astype(np.float64)
    th = pose[:, 2].astype(np.float64)
    v = np.where(meta[:, 2] != 0, 0.0, goal[:, 2].astype(np.float64))
    return p, th, np.stack((v * np.cos(th), v * np.sin(th)), 1)


def _rot(e, a):
    c, s = np.cos(a), np.sin(a)
    return np.array([c * e[0] - s * e[1], s * e[0] + c * e[1]])


def half_plane(pa, va, pb, vb, r, tau, dt):
    """ORCA half-plane of agent a against b as (P, n): allowed velocities v have (v - P) . n >= 0.  None when the
    relative velocity is the centre of the one-step disk (no outward direction)."""
    rp = pb - pa
    rv = va - vb
    dist = float(np.hypot(*rp))
    if dist > r:
        c, R = rp / tau, r / tau
        cands = []
        w = rv - c
        wl = float(np.hypot(*w))
        if wl > 0:
            m = w / wl
            if float(m @ (-rp / dist)) >= r / dist:          # radial projection lands on the cap arc
                cands.append((abs(wl - R), c + R * m, m))
        alpha = np.arcsin(r / dist)
        tangent = np.sqrt(dist * dist - r * r) / tau           # apex -> tangent point
        for side in (1.0, -1.0):
            e = _rot(rp / dist, side * alpha)
            q = max(float(rv @ e), tangent) * e
            n = np.array([-e[1], e[0]]) if side > 0 else np.array([e[1], -e[0]])
            cands.append((float(np.hypot(*(q - rv))), q, n))
        _, q, n = min(cands, key=lambda t: t[0])
    else:
        c, R = rp / dt, r / dt
        w = rv - c
        wl = float(np.hypot(*w))
        if wl == 0.0:
            return None
        n = w / wl
        q = c + R * n
    return va + 0.5 * (q - rv), n


def penetration(P, n, v):
    """Penetration of velocity v into each half-plane (> 0 = violated)."""
    return ((P - np.asarray(v, np.float64)) * n).sum(-1)


def _line_circle(a, b, rad):
    """Points v with a . v = b and |v| = rad, for rows of a (k, 2) / b (k)."""
    aa = (a * a).sum(1)
    ok = aa > 1e-24
    a, b, aa = a[ok], b[ok], aa[ok]
    foot = a * (b / aa)[:, None]
    h2 = rad * rad - (foot * foot).sum(1)
    keep = h2 >= 0
    foot, a, aa, h = foot[keep], a[keep], aa[keep], np.sqrt(h2[keep])
    perp = np.stack((-a[:, 1], a[:, 0]), 1) / np.sqrt(aa)[:, None]
    return np.concatenate((foot + perp * h[:, None], foot - perp * h[:, None]))


@lru_cache(maxsize=None)
def _combinations(k, m):
    """Index arrays (m, C(k, m)) of every m-subset of range(k), in itertools order."""
    return np.array(list(combinations(range(k), m)), np.intp).reshape(-1, m).T


def _solve2(a1, b1, a2, b2):
    det = a1[:, 0] * a2[:, 1] - a1[:, 1] * a2[:, 0]
    ok = np.abs(det) > 1e-12
    a1, b1, a2, b2, det = a1[ok], b1[ok], a2[ok], b2[ok], det[ok]
    return np.stack(((b1 * a2[:, 1] - b2 * a1[:, 1]) / det, (a1[:, 0] * b2 - a2[:, 0] * b1) / det), 1)


def project(P, n, vmax, vpref):
    """argmin |v - vpref| over the half-planes and |v| <= vmax, or None when they have no common point."""
    vpref = np.asarray(vpref, np.float64)
    c = (P * n).sum(1)                                      # boundary of line i: n_i . v = c_i
    cands = [vpref[None]]
    nv = float(np.hypot(*vpref))
    if nv > 0:
        cands.append((vpref * (vmax / nv))[None])
    if len(c):
        cands.append(vpref[None] + penetration(P, n, vpref)[:, None] * n)
        cands.append(_line_circle(n, c, vmax))
        if len(c) > 1:
            i, j = _combinations(len(c), 2)
            cands.append(_solve2(n[i], c[i], n[j], c[j]))
    v = np.concatenate(cands)
    ok = np.hypot(v[:, 0], v[:, 1]) <= vmax + FEAS_TOL
    if len(c):
        ok &= (c[None, :] - v @ n.T).max(1) <= FEAS_TOL
    if not ok.any():
        return None
    v = v[ok]
    return v[np.argmin(np.hypot(v[:, 0] - vpref[0], v[:, 1] - vpref[1]))]


def min_max_penetration(P, n, vmax):
    """min over |v| <= vmax of the largest penetration, and a minimiser.  The optimum of a maximum of linear functions
    on a disk lies where one function is least on the circle, where two are equal on the circle, or where three are
    equal."""
    c = (P * n).sum(1)
    k = len(c)
    cands = [vmax * n]
    if k > 1:
        i, j = _combinations(k, 2)
        cands.append(_line_circle(n[j] - n[i], c[j] - c[i], vmax))
    if k > 2:
        i, j, l = _combinations(k, 3)
        cands.append(_solve2(n[j] - n[i], c[j] - c[i], n[l] - n[i], c[l] - c[i]))
    v = np.concatenate(cands)
    v = v[np.hypot(v[:, 0], v[:, 1]) <= vmax + FEAS_TOL]
    g = (c[None, :] - v @ n.T).max(1)
    b = int(np.argmin(g))
    return float(g[b]), v[b]


def preferred(p, goal, vmax, dt):
    d = np.asarray(goal, np.float64) - p
    dl = float(np.hypot(*d))
    return np.zeros(2) if dl == 0 else d * min(vmax / dl, 1.0 / dt)


def track(th, v, vmax, wmin, wmax, gain):
    """Heading tracker: ORCA velocity -> raw (v, w)."""
    nrm = float(np.hypot(*v))
    if nrm <= 1e-6:
        return np.zeros(2)
    c = v[0] * np.cos(th) + v[1] * np.sin(th)
    s = v[1] * np.cos(th) - v[0] * np.sin(th)
    if c > 0:
        return np.array([min(c, vmax), min(max(gain * s / nrm, wmin), wmax)])
    return np.array([0.0, wmax if s >= 0 else wmin])


def agent_lines(pose, goal, meta, R, a, radius, neighbour_dist, tau, dt):
    """Half-planes (P (k, 2), n (k, 2)) of agent a from the other robots of its world within neighbour_dist."""
    p, _, vel = agent_state(pose, goal, meta)
    base = a - a % R
    Ps, ns = [], []
    for b in range(base, base + R):
        if b == a or np.hypot(*(p[b] - p[a])) >= neighbour_dist:
            continue
        hp = half_plane(p[a], vel[a], p[b], vel[b], 2.0 * radius, tau, dt)
        if hp is not None:
            Ps.append(hp[0])
            ns.append(hp[1])
    return np.array(Ps).reshape(-1, 2), np.array(ns).reshape(-1, 2)
