"""Numpy restatement of the arena layout of csrc/rlca_layout.cu (DESIGN.md §9v), written from the rule: the arena of a
world (pick 0: global world mod T; pick 1: (m T) >> 24 of the draw (agent0, episode, 0, 0xA0)), try k of a start or goal
a uniform cell of the arena's list ((m n_a) >> 24 of the draw (agent, episode, k, 0xA3 / 0xA4)) and a uniform point of
that cell, the first accepted try per robot, float32 arithmetic one rounding per operation.  Philox, the heading and
pre_distance come from layout_ref."""
import numpy as np

import layout_ref

_F = np.float32
PURPOSE_ARENA = 0xA0


def _m24(u):
    """The 24-bit integer m = 2^24 u of uniforms u."""
    return (np.asarray(u, np.float64) * 2.0 ** 24).astype(np.uint64)


def arena_of(seed, agent0, episode, pick, world, T):
    if pick == 0:
        return world % T
    u = layout_ref.rand4(seed, agent0, episode, [0], PURPOSE_ARENA)
    return int((_m24(u[0])[0] * np.uint64(T)) >> np.uint64(24))


def draws(seed, agent, episode, ks, purpose, cells, ocx, ocy, res):
    """(x, y, cell index) of tries ks of one robot in an arena whose cells are `cells` (packed)."""
    u = layout_ref.rand4(seed, agent, episode, ks, PURPOSE_ARENA | purpose)
    idx = (_m24(u[0]) * np.uint64(len(cells))) >> np.uint64(24)
    c = cells[idx.astype(np.int64)].astype(np.int64)
    x = (((c & 0xFFFF) - ocx).astype(_F) + u[1]) * _F(res)
    y = (((c >> 16) - ocy).astype(_F) + u[2]) * _F(res)
    return x.astype(_F), y.astype(_F), idx.astype(np.int64)


def _first_accept(seed, agent, episode, purpose, max_reject, ok_fn, arena, chunk=64):
    for base in range(0, max_reject, chunk):
        ks = np.arange(base, min(base + chunk, max_reject))
        x, y, _ = draws(seed, agent, episode, ks, purpose, *arena)
        hit = np.flatnonzero(ok_fn(x, y))
        if len(hit):
            return int(ks[hit[0]]), x[hit[0]], y[hit[0]]
    return None


def world_layout(cfg, sep2, tr2, tables, pick, w, episode):
    """(a, sx, sy, gx, gy, th, tries) of world w at `episode`, or (a, 1 + r, tries) when robot r is not placed; `tries`
    (R, 2) holds the accepted try of each start and goal, -1 unplaced."""
    R, seed, mr = int(cfg.robots_per_world), int(cfg.seed), int(cfg.max_reject)
    world = int(cfg.world_offset) + w
    agent0 = (world * R) & 0xFFFFFFFF
    a = arena_of(seed, agent0, episode, pick, world, tables.count)
    arena = (tables.cells[tables.cell_off[a]:tables.cell_off[a + 1]], int(cfg.origin_cx), int(cfg.origin_cy),
             _F(cfg.resolution))
    sx, sy, gx, gy = (np.zeros(0, _F) for _ in range(4))
    tries = np.full((R, 2), -1, np.int64)
    for r in range(R):
        ag = (agent0 + r) & 0xFFFFFFFF
        s = _first_accept(seed, ag, episode, 3, mr, lambda x, y: layout_ref._far(x, y, sx, sy, sep2), arena)
        if s is None:
            return a, 1 + r, tries
        tries[r, 0], x0, y0 = s
        sx, sy = np.append(sx, x0), np.append(sy, y0)
        g = _first_accept(seed, ag, episode, 4, mr, lambda x, y: layout_ref._far(x, y, _F([x0]), _F([y0]), tr2)
                          & layout_ref._far(x, y, gx, gy, sep2), arena)
        if g is None:
            return a, 1 + r, tries
        tries[r, 1] = g[0]
        gx, gy = np.append(gx, g[1]), np.append(gy, g[2])
    th = [layout_ref.normalize(layout_ref.rand4(seed, (agent0 + r) & 0xFFFFFFFF, episode, [0], 5)[0, 0] *
                               layout_ref.TWO_PI_F) for r in range(R)]
    return a, sx, sy, gx, gy, th, tries


def _pre_distance(cfg, sx, sy, gx, gy):
    if cfg.pre_distance_zero:
        return _F(0.0)
    ddx, ddy = _F(gx - sx), _F(gy - sy)
    return np.sqrt(layout_ref.fmaf(ddx, ddx, _F(ddy * ddy)))


def layout(cfg, lay, pick, pose, goal, acc):
    """rlca_layout_arena_host restated.  Returns (pose, goal, acc, status, arenas (W,), tries (W, R, 2))."""
    R, W = int(cfg.robots_per_world), int(cfg.num_worlds)
    sep2, tr2 = _F(lay.separation) * _F(lay.separation), _F(lay.min_travel) * _F(lay.min_travel)
    pose, goal, acc = (np.array(a, _F, copy=True) for a in (pose, goal, acc))
    status = np.zeros(W, np.int32)
    arenas = np.zeros(W, np.int64)
    tries = np.full((W, R, 2), -1, np.int64)
    for w in range(W):
        res = world_layout(cfg, sep2, tr2, lay.tables, pick, w, 0)
        arenas[w], tries[w] = res[0], res[-1]
        if len(res) == 3:
            status[w] = res[1]
            continue
        _, sx, sy, gx, gy, th, _ = res
        for r in range(R):
            i = w * R + r
            pose[i, 0:3] = sx[r], sy[r], th[r]
            pose[i, 3] = _pre_distance(cfg, sx[r], sy[r], gx[r], gy[r])
            goal[i, 0:2] = gx[r], gy[r]
            acc[i, 2:4] = sx[r], sy[r]
    return pose, goal, acc, status, arenas, tries


def relayout(cfg, lay, pick, pose, goal, acc, meta, flags):
    """rlca_layout_arena_respawn_host restated: latched robots parked, a world whose robots are all latched re-laid in
    its arena at episode meta.y + 1 and written as a new episode.  Returns (pose, goal, acc, meta, flags, live,
    status)."""
    R, W = int(cfg.robots_per_world), int(cfg.num_worlds)
    sep2, tr2 = _F(lay.separation) * _F(lay.separation), _F(lay.min_travel) * _F(lay.min_travel)
    pose, goal, acc = (np.array(a, _F, copy=True) for a in (pose, goal, acc))
    meta, flags = np.array(meta, np.int32, copy=True), np.array(flags, np.uint8, copy=True)
    live = np.zeros(R * W, np.uint8)
    status = np.zeros(W, np.int32)
    for w in range(W):
        rows = slice(w * R, (w + 1) * R)
        latched = meta[rows, 3] != 0
        if latched.all():
            e = int(meta[w * R, 1]) + 1
            res = world_layout(cfg, sep2, tr2, lay.tables, pick, w, e & 0xFFFFFFFF)
            if len(res) == 7:
                _, sx, sy, gx, gy, th, _ = res
                for r in range(R):
                    i = w * R + r
                    pose[i, 0:3] = sx[r], sy[r], th[r]
                    pose[i, 3] = _pre_distance(cfg, sx[r], sy[r], gx[r], gy[r])
                    goal[i] = gx[r], gy[r], 0.0, 0.0
                    acc[i, 0] = 0.0
                    acc[i, 2:4] = sx[r], sy[r]
                    meta[i, 0], meta[i, 1], meta[i, 3] = 1, e, 0
                    flags[i, 3] = 1
                live[rows] = 1
                continue
            status[w] = res[1]
        goal[w * R:(w + 1) * R][latched, 2:4] = 0.0
        live[rows] = (~latched).astype(np.uint8)
    return pose, goal, acc, meta, flags, live, status
