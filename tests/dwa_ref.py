"""Float64 restatement of the dynamic-window baseline (DESIGN.md §9u, csrc/rlca_dwa.cu), written from the algorithm
and not from the kernel: every return of the newest frame is used (no reach filter), beam directions are the exact
angles, and each candidate's clearance is the minimum over all points of the closed-form contact arc length."""
import math

import numpy as np

STRAIGHT_W = 1e-6


def beam_angles(cfg):
    """Exact beam angles of the env's nearest-index sub-sampling of the raw beams (its running sums restated)."""
    raw, nb = int(cfg.raw_beams), int(cfg.beams)
    step, half = raw / nb, nb // 2
    index, out = 0.0, [0] * nb
    for i in range(half):
        out[i] = int(index)
        index += step
    index = raw - 1.0
    for i in range(half):
        out[nb - 1 - i] = int(index)
        index -= step
    fov = float(cfg.fov)
    return -0.5 * fov + np.asarray(out, np.float64) * (fov / (raw - 1))


def window(cfg, p, v0, w0):
    v0 = min(max(v0, cfg.v_min), cfg.v_max)
    w0 = min(max(w0, cfg.w_min), cfg.w_max)
    adt, aadt = p.accel * cfg.dt, p.angular_accel * cfg.dt
    v_lo, v_hi = (max(cfg.v_min, v0 - adt), min(cfg.v_max, v0 + adt)) if adt > 0 else (cfg.v_min, cfg.v_max)
    w_lo, w_hi = (max(cfg.w_min, w0 - aadt), min(cfg.w_max, w0 + aadt)) if aadt > 0 else (cfg.w_min, cfg.w_max)
    samp = lambda lo, hi, n: np.array([0.5 * (lo + hi)]) if n == 1 else lo + (hi - lo) * np.arange(n) / (n - 1)
    v, w = samp(v_lo, v_hi, p.v_samples), samp(w_lo, w_hi, p.w_samples)
    return np.repeat(v, p.w_samples), np.tile(w, p.v_samples), (v_lo, v_hi, w_lo, w_hi)


def contact(v, w, px, py, rho):
    """Arc length to the first contact of the disc on the (v, w) path with each point (px, py), +inf without one;
    v > 0, points at least rho from the robot."""
    if abs(w) < STRAIGHT_W:
        hit = (px > 0) & (np.abs(py) < rho)
        return np.where(hit, np.maximum(px - np.sqrt(np.maximum(rho * rho - py * py, 0.0)), 0.0), np.inf)
    R = v / abs(w)
    y = -py if w < 0 else py
    D = np.hypot(px, y - R)
    hit = np.abs(D - R) < rho
    cosa = np.clip((R * R + D * D - rho * rho) / (2 * R * D), -1.0, 1.0)
    alpha = np.arccos(cosa)
    th = np.arctan2(px, R - y) % (2 * math.pi)
    return np.where(hit, R * np.maximum(th - alpha, 0.0), np.inf)


def contact_sampled(v, w, px, py, rho, length, step):
    """Brute force: the first arc length, on a grid of `step`, at which the disc centre comes within rho of the point
    (inf when it does not within `length`)."""
    s = np.arange(0.0, length + step, step)
    if abs(w) < STRAIGHT_W:
        cx, cy = s, np.zeros_like(s)
    else:
        th = s * w / v
        R = v / w
        cx, cy = R * np.sin(th), R * (1 - np.cos(th))
    d = np.hypot(cx - px, cy - py)
    inside = np.flatnonzero(d < rho)
    return s[inside[0]] if len(inside) else math.inf


def robot(cfg, p, scan, gs, cap):
    """One robot: (v, w, clearance, admissibility margin, score) per candidate, float64."""
    r = (scan.astype(np.float64) + 0.5) * cfg.range_max
    ret = r < np.float32(cfg.range_max)
    b = beam_angles(cfg)
    px, py = (r * np.cos(b))[ret], (r * np.sin(b))[ret]
    touch = bool((r[ret] < p.radius).any())
    vs, ws, _ = window(cfg, p, float(gs[2]), float(gs[3]))
    out = []
    for v, w in zip(vs, ws):
        if touch:
            cl = 0.0
        elif v == 0:
            cl = cap
        else:
            cl = min(v * p.horizon, float(contact(v, w, px, py, p.radius).min(initial=math.inf)))
        need = v * cfg.dt + v * v / (2 * p.brake)
        margin = cl - need                  # admissible iff cl > 0 and margin >= 0
        T = p.heading_time
        if v == 0:
            hx, hy, th = 0.0, 0.0, w * T
        elif abs(w) < STRAIGHT_W:
            hx, hy, th = v * T, 0.0, 0.0
        else:
            th = w * T
            hx, hy = v / w * math.sin(th), v / w * (1 - math.cos(th))
        dx, dy = gs[0] - hx, gs[1] - hy
        bearing = math.atan2(dy * math.cos(th) - dx * math.sin(th), dx * math.cos(th) + dy * math.sin(th))
        score = p.heading_weight * (1 - abs(bearing) / math.pi) + p.clearance_weight * min(cl, cap) / cap + \
            p.speed_weight * v / cfg.v_max
        out.append((v, w, cl, margin, score))
    return np.array(out)
