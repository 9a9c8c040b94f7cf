"""Numpy restatement of the arena curriculum of csrc/rlca_layout.cu (DESIGN.md §9z), written from the rule: the fold
E = decay E + e, S = decay S + s, p = (S + 1) / (E + 2), q = uniform + (1 - uniform) 4 p (1 - p), w = max(1,
floor(2^20 q)) in float32 with one rounding per operation, the cdf the exclusive prefix sum of w; the weighted arena
a with cdf[a] <= (m cdf[T]) >> 24 < cdf[a + 1] for pick 1's m; the tally of a tick's ended, unmasked rows against the
arena a world held before its re-layout.  Starts, goals and headings come from arena_ref and layout_ref."""
import numpy as np

import arena_ref
import layout_ref

_F = np.float32
ONE = 1 << 20


def fold(E, S, pending, decay, uniform):
    """(E, S, weights (T,) uint64, cdf (T + 1,) uint64) after one update."""
    E, S = np.asarray(E, _F), np.asarray(S, _F)
    T = len(E)
    pending = np.asarray(pending, np.int32)
    d, u = _F(decay), _F(uniform)
    E = d * E + pending[:T].astype(_F)
    S = d * S + pending[T:].astype(_F)
    p = (S + _F(1)) / (E + _F(2))
    q = u + (_F(1) - u) * (_F(4) * p * (_F(1) - p))
    v = q * _F(ONE)
    w = np.where(v >= _F(ONE), ONE, np.where(v >= _F(1), np.floor(v), 1)).astype(np.uint64)
    cdf = np.zeros(T + 1, np.uint64)
    cdf[1:] = np.cumsum(w, dtype=np.uint64)
    return E.astype(_F), S.astype(_F), w, cdf


def weighted_arena(seed, agent0, episode, cdf):
    u = layout_ref.rand4(seed, agent0, episode, [0], arena_ref.PURPOSE_ARENA)
    m = int(np.float64(u[0][0]) * 2.0 ** 24)
    target = (m * int(cdf[-1])) >> 24
    return int(np.searchsorted(np.asarray(cdf[:-1], np.uint64), np.uint64(target), side='right')) - 1


def world_layout(cfg, sep2, tr2, tables, cdf, w, episode):
    """arena_ref.world_layout with the weighted arena: (a, sx, sy, gx, gy, th) of world w, or (a, 1 + r)."""
    R, seed, mr = int(cfg.robots_per_world), int(cfg.seed), int(cfg.max_reject)
    agent0 = ((int(cfg.world_offset) + w) * R) & 0xFFFFFFFF
    a = weighted_arena(seed, agent0, episode, cdf)
    arena = (tables.cells[tables.cell_off[a]:tables.cell_off[a + 1]], int(cfg.origin_cx), int(cfg.origin_cy),
             _F(cfg.resolution))
    sx, sy, gx, gy = (np.zeros(0, _F) for _ in range(4))
    for r in range(R):
        ag = (agent0 + r) & 0xFFFFFFFF
        s = arena_ref._first_accept(seed, ag, episode, 3, mr, lambda x, y: layout_ref._far(x, y, sx, sy, sep2), arena)
        if s is None:
            return a, 1 + r
        _, x0, y0 = s
        sx, sy = np.append(sx, x0), np.append(sy, y0)
        g = arena_ref._first_accept(seed, ag, episode, 4, mr, lambda x, y: layout_ref._far(x, y, _F([x0]), _F([y0]), tr2)
                                    & layout_ref._far(x, y, gx, gy, sep2), arena)
        if g is None:
            return a, 1 + r
        gx, gy = np.append(gx, g[1]), np.append(gy, g[2])
    th = [layout_ref.normalize(layout_ref.rand4(seed, (agent0 + r) & 0xFFFFFFFF, episode, [0], 5)[0, 0] *
                               layout_ref.TWO_PI_F) for r in range(R)]
    return a, sx, sy, gx, gy, th


def _consts(cfg, lay):
    return _F(lay.separation) * _F(lay.separation), _F(lay.min_travel) * _F(lay.min_travel)


def layout(cfg, lay, cdf, world_arena, pose, goal, acc):
    """rlca_layout_arena_weighted_host restated: (pose, goal, acc, status, world_arena)."""
    R, W = int(cfg.robots_per_world), int(cfg.num_worlds)
    sep2, tr2 = _consts(cfg, lay)
    pose, goal, acc = (np.array(a, _F, copy=True) for a in (pose, goal, acc))
    world_arena = np.array(world_arena, np.int32, copy=True)
    status = np.zeros(W, np.int32)
    for w in range(W):
        res = world_layout(cfg, sep2, tr2, lay.tables, cdf, w, 0)
        if len(res) == 2:
            status[w] = res[1]
            continue
        a, sx, sy, gx, gy, th = res
        world_arena[w] = a
        for r in range(R):
            i = w * R + r
            pose[i, 0:3] = sx[r], sy[r], th[r]
            pose[i, 3] = arena_ref._pre_distance(cfg, sx[r], sy[r], gx[r], gy[r])
            goal[i, 0:2] = gx[r], gy[r]
            acc[i, 2:4] = sx[r], sy[r]
    return pose, goal, acc, status, world_arena


def tally(flags, row_mask, world_arena, pending, R):
    """pending after the tally of one tick's flags (N, 4) against world_arena."""
    f = np.asarray(flags, np.uint8)
    ended = (f[:, 0] != 0) & (f[:, 2] != 0)
    if row_mask is not None:
        ended &= np.asarray(row_mask) == 0
    reached = ended & (f[:, 2] == 1)
    pending = np.array(pending, np.int32, copy=True)
    T = len(pending) // 2
    for w, a in enumerate(world_arena):
        e, s = int(ended[w * R:(w + 1) * R].sum()), int(reached[w * R:(w + 1) * R].sum())
        if e and 0 <= a < T:
            pending[a] += e
            pending[T + a] += s
    return pending


def relayout(cfg, lay, cdf, world_arena, pending, row_mask, pose, goal, acc, meta, flags):
    """rlca_layout_arena_weighted_respawn_host restated: (pose, goal, acc, meta, flags, live, status, world_arena,
    pending)."""
    R, W = int(cfg.robots_per_world), int(cfg.num_worlds)
    sep2, tr2 = _consts(cfg, lay)
    pending = tally(flags, row_mask, world_arena, pending, R)
    pose, goal, acc = (np.array(a, _F, copy=True) for a in (pose, goal, acc))
    meta, flags = np.array(meta, np.int32, copy=True), np.array(flags, np.uint8, copy=True)
    world_arena = np.array(world_arena, np.int32, copy=True)
    live = np.zeros(R * W, np.uint8)
    status = np.zeros(W, np.int32)
    for w in range(W):
        rows = slice(w * R, (w + 1) * R)
        latched = meta[rows, 3] != 0
        if latched.all():
            e = int(meta[w * R, 1]) + 1
            res = world_layout(cfg, sep2, tr2, lay.tables, cdf, w, e & 0xFFFFFFFF)
            if len(res) == 6:
                a, sx, sy, gx, gy, th = res
                world_arena[w] = a
                for r in range(R):
                    i = w * R + r
                    pose[i, 0:3] = sx[r], sy[r], th[r]
                    pose[i, 3] = arena_ref._pre_distance(cfg, sx[r], sy[r], gx[r], gy[r])
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
    return pose, goal, acc, meta, flags, live, status, world_arena, pending
