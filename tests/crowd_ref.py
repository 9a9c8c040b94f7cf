"""Float64 restatement of the social-force crowd (DESIGN.md §9t), from the definition: the driving term towards the
§9h driver's preferred velocity, the anisotropic agent repulsion with its sideways bias, the wall repulsion from every
boundary segment within wall_dist with the agent on its free side, one Euler step on the speed disk and ORCA-DD's
heading tracker.  Nothing here follows the kernel's lane order or its bin lists: walls are all segments of the set."""
from __future__ import annotations

import numpy as np

import orca_ref


def wall_terms(p, segments, wall_dist):
    """(distance d, unit n = (p - q) / d) of every segment (x0, y0, x1, y1) closer than wall_dist with p strictly on its
    right (free) side and d > 0."""
    out = []
    for x0, y0, x1, y1 in np.asarray(segments, np.float64):
        a, e = np.array([x0, y0]), np.array([x1 - x0, y1 - y0])
        t = min(max(float((p - a) @ e) / float(e @ e), 0.0), 1.0)
        q = a + t * e
        d = float(np.hypot(*(p - q)))
        free = e[0] * (p - a)[1] - e[1] * (p - a)[0] < 0.0
        if free and 0.0 < d < wall_dist:
            out.append((d, (p - q) / d))
    return out


def crowd_action(cfg, pose, goal, meta, mask, a, params, segments=None):
    """The action of crowd agent a (float64 (v, w)); `params` a crowd.CrowdParams, `segments` (S, 4) or None."""
    R = cfg.robots_per_world
    pos, th, vel = orca_ref.agent_state(pose, goal, meta)
    speed = float(cfg.v_max) if params.speed is None else float(params.speed)
    u0 = orca_ref.preferred(pos[a], goal[a, 0:2].astype(np.float64), speed, float(cfg.dt))
    f = (u0 - vel[a]) / params.relax_time
    h = np.array([np.cos(th[a]), np.sin(th[a])])
    lam = params.anisotropy
    base = a - a % R
    for j in range(base, base + R):
        if j == a or not (params.see_robots or mask[j]):
            continue
        d = float(np.hypot(*(pos[a] - pos[j])))
        if not 0.0 < d < params.neighbour_dist:
            continue
        n = (pos[a] - pos[j]) / d
        t = np.array([-n[1], n[0]])
        w = lam + (1.0 - lam) * (1.0 + float(-n @ h)) / 2.0
        f = f + params.strength * np.exp((2.0 * params.radius - d) / params.range) * w * (n + params.side_bias * t)
    if segments is not None:
        for d, n in wall_terms(pos[a], segments, params.wall_dist):
            f = f + params.wall_strength * np.exp((params.radius - d) / params.wall_range) * n
    u = vel[a] + f * float(cfg.dt)
    un = float(np.hypot(*u))
    if un > speed:
        u = u * (speed / un)
    return orca_ref.track(th[a], u, speed, float(cfg.w_min), float(cfg.w_max), params.heading_gain)


def distances(cfg, pose, a, segments=None, wall_dist=None):
    """Agent a's distances to the other agents of its world and, with segments, to every segment with a on its free
    side: what the cut-offs compare."""
    R = cfg.robots_per_world
    p = pose[:, 0:2].astype(np.float64)
    base = a - a % R
    ds = [float(np.hypot(*(p[a] - p[j]))) for j in range(base, base + R) if j != a]
    if segments is not None:
        ds += [d for d, _ in wall_terms(p[a], segments, np.inf)]
    return np.array(ds)
