"""Float64 reference of the NH-ORCA controller (DESIGN.md §9e), written from the definition (Alonso-Mora, Breitenmoser,
Rufli, Beardsley, Siegwart, "Optimal reciprocal collision avoidance for multiple non-holonomic robots", DARS 2010):

- the tracking error of an arc, by following the unicycle over dense t and measuring its distance from the holonomic
  trajectory, not from the closed form V T_th |sin(th/2)|;
- the speed bound V_max(th) of the velocity set S_E;
- the LP with P's edges as hard lines: orca_ref.project with P's half-planes appended as extra rows;
- the least-penetration fallback: min t subject to every ORCA penetration <= t and u in P, an exact LP
  (scipy.optimize.linprog; P lies inside the speed disk, so the disk is redundant);
- the arc tracker.

Nothing here follows the structure of the CUDA code.
"""
from __future__ import annotations

import numpy as np
from scipy.optimize import linprog

import orca_ref


def turn_time(th, T, wmin, wmax):
    """T_th = max(T, th / w_max) for th >= 0, max(T, th / w_min) for th < 0."""
    th = np.asarray(th, np.float64)
    return np.where(th >= 0, np.maximum(T, th / wmax), np.maximum(T, th / wmin))


def arc_speed(V, th):
    """v* = V (th/2) cot(th/2), V at th = 0."""
    th = np.asarray(th, np.float64)
    h = 0.5 * th
    with np.errstate(invalid='ignore', divide='ignore'):
        return np.where(h == 0, V, V * h * np.cos(h) / np.sin(h))


def speed_bound(th, E, T, vmax, wmin, wmax):
    """V_max(th) = min(v_max, E / (T_th |sin(th/2)|))."""
    th = np.asarray(th, np.float64)
    s = np.abs(np.sin(0.5 * th))
    with np.errstate(divide='ignore'):
        return np.minimum(vmax, np.where(s > 0, E / (turn_time(th, T, wmin, wmax) * s), np.inf))


def deviation(v, w, turn, V, th, steps=2001, after=1.0):
    """Largest distance between the unicycle that drives at (v, w) for `turn` s and then straight at V, and the
    holonomic point V t (cos th, sin th), over t in [0, turn + after] on `steps` points per phase.  The unicycle is
    followed by summing its exact arcs between the grid points, from the heading at each one."""
    t1 = np.linspace(0.0, turn, steps)
    dt = np.diff(t1)
    head = w * t1
    # exact arc between t_k and t_k+1 at constant (v, w)
    if w != 0:
        dx = v / w * (np.sin(head[1:]) - np.sin(head[:-1]))
        dy = v / w * (np.cos(head[:-1]) - np.cos(head[1:]))
    else:
        dx, dy = v * dt, np.zeros_like(dt)
    x = np.concatenate(([0.0], np.cumsum(dx)))
    y = np.concatenate(([0.0], np.cumsum(dy)))
    t2 = np.linspace(0.0, after, steps)[1:]
    hend = head[-1]
    x = np.concatenate((x, x[-1] + V * t2 * np.cos(hend)))
    y = np.concatenate((y, y[-1] + V * t2 * np.sin(hend)))
    t = np.concatenate((t1, turn + t2))
    return float(np.hypot(x - V * t * np.cos(th), y - V * t * np.sin(th)).max())


def tracking_error(V, th, T, wmin, wmax, steps=2001):
    """epsilon(V, th): the largest distance of the arc tracker (v*, th / T_th for T_th, then straight) from the
    holonomic trajectory, measured."""
    turn = float(turn_time(th, T, wmin, wmax))
    return deviation(float(arc_speed(V, th)), th / turn, turn, V, th, steps)


def polygon_half_planes(verts, heading):
    """P's edges rotated by `heading` as half-planes (P (k, 2), n (k, 2)): (v - P) . n >= 0 inside."""
    c, s = np.cos(heading), np.sin(heading)
    rot = np.array([[c, -s], [s, c]])
    v = verts.astype(np.float64) @ rot.T
    d = np.roll(v, -1, axis=0) - v
    n = np.stack((-d[:, 1], d[:, 0]), 1)
    return v, n / np.hypot(n[:, 0], n[:, 1])[:, None]


def project(P, n, Ph, nh, vmax, vpref):
    """argmin |u - v_pref| over the ORCA half-planes, P and |u| <= v_max, or None."""
    return orca_ref.project(np.concatenate((Ph, P)), np.concatenate((nh, n)), vmax, vpref)


def least_penetration(P, n, Ph, nh):
    """(t*, u*): min over u in P of the largest penetration into the ORCA half-planes."""
    k = len(n)
    # variables (ux, uy, t): c_j - n_j . u <= t for the ORCA lines, c_h - n_h . u <= 0 for P
    A = np.concatenate((np.concatenate((-n, -np.ones((k, 1))), 1), np.concatenate((-nh, np.zeros((len(nh), 1))), 1)))
    b = np.concatenate((-(P * n).sum(1), -(Ph * nh).sum(1)))
    res = linprog([0.0, 0.0, 1.0], A_ub=A, b_ub=b, bounds=[(None, None)] * 3, method='highs')
    assert res.status == 0, res.message
    return float(res.x[2]), res.x[:2]


def track(heading, u, vmin, vmax, wmin, wmax, T):
    """The arc tracker: world-frame velocity u -> raw (v, w), and (V, th, T_th)."""
    V = float(np.hypot(*u))
    if V <= 1e-6:
        return np.zeros(2), (V, 0.0, T)
    c = u[0] * np.cos(heading) + u[1] * np.sin(heading)
    s = u[1] * np.cos(heading) - u[0] * np.sin(heading)
    th = float(np.arctan2(s, c))
    turn = float(turn_time(th, T, wmin, wmax))
    v = float(arc_speed(V, th))
    return np.array([min(max(v, vmin), vmax), min(max(th / turn, wmin), wmax)]), (V, th, turn)
