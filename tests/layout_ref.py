"""Numpy restatement of the random layout of csrc/rlca_layout.cu (DESIGN.md §9i), written from the rule, not the code:
Philox-4x32-10 in uint64 arithmetic, the first accepted try per robot, float32 arithmetic one rounding per operation.
pre_distance (only when pre_distance_zero is 0) rounds fmaf exactly through rationals."""
from fractions import Fraction

import numpy as np

_MASK = np.uint64(0xFFFFFFFF)
_F = np.float32
TWO_PI_F = _F(6.28318548202514648438)
PI_F = _F(3.14159274101257324219)


def philox(c, k0, k1):
    """Philox-4x32-10 of the counters c (4 arrays of uint32 values) under the key (k0, k1)."""
    c0, c1, c2, c3 = (np.asarray(x, np.uint64) & _MASK for x in c)
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
        k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK
        k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK
    return c0, c1, c2, c3


def rand4(seed, agent, episode, draws, purpose):
    """(4, len(draws)) float32 uniforms: the top 24 bits of each Philox word times 2^-24."""
    d = np.asarray(draws, np.uint64)
    n = d.shape[0]
    full = lambda v: np.full(n, v, np.uint64)
    out = philox((full(agent), full(episode), d, full(purpose)), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    return np.stack([(w >> np.uint64(8)).astype(np.float32) * _F(2.0 ** -24) for w in out])


def normalize(a):
    a = _F(a)
    if a > PI_F:
        return _F(a - TWO_PI_F)
    if a <= -PI_F:
        return _F(a + TWO_PI_F)
    return a


def _round_f32(q):
    """The float32 nearest to the rational q, ties to even."""
    f = _F(float(q))
    cands = [np.nextafter(f, _F(-np.inf)), f, np.nextafter(f, _F(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1))


def fmaf(a, b, c):
    return _round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _first_accept(seed, agent, purpose, side, max_reject, ok_fn, chunk=64):
    """(k, x, y) of the first try k < max_reject whose draw ok_fn accepts, or None."""
    for base in range(0, max_reject, chunk):
        ks = np.arange(base, min(base + chunk, max_reject))
        u = rand4(seed, agent, 0, ks, purpose)
        x = (u[0] - _F(0.5)) * _F(side)
        y = (u[1] - _F(0.5)) * _F(side)
        hit = np.flatnonzero(ok_fn(x, y))
        if len(hit):
            i = hit[0]
            return int(ks[i]), x[i], y[i]
    return None


def _far(x, y, px, py, d2):
    """(tries,) True where the draw is at least sqrt(d2) from every point (px, py), squared distances in float32."""
    if len(px) == 0:
        return np.ones(x.shape, bool)
    dx = x[:, None] - px[None, :]
    dy = y[:, None] - py[None, :]
    return (dx * dx + dy * dy >= d2).all(1)


def layout(cfg, side, separation, min_travel, pose, goal, acc):
    """The layout of every world of cfg written into copies of pose, goal, acc (N, 4).  Returns (pose, goal, acc,
    status (num_worlds,) int32, tries (num_worlds, R, 2) the accepted try index of each start and goal, -1 unplaced)."""
    R, W = int(cfg.robots_per_world), int(cfg.num_worlds)
    seed, mr = int(cfg.seed), int(cfg.max_reject)
    sep2 = _F(separation) * _F(separation)
    tr2 = _F(min_travel) * _F(min_travel)
    pose, goal, acc = (np.array(a, np.float32, copy=True) for a in (pose, goal, acc))
    status = np.zeros(W, np.int32)
    tries = np.full((W, R, 2), -1, np.int64)
    for w in range(W):
        agent0 = ((int(cfg.world_offset) + w) * R) & 0xFFFFFFFF
        sx, sy, gx, gy = (np.zeros(0, np.float32) for _ in range(4))
        for r in range(R):
            a = (agent0 + r) & 0xFFFFFFFF
            s = _first_accept(seed, a, 3, side, mr, lambda x, y: _far(x, y, sx, sy, sep2))
            if s is None:
                status[w] = 1 + r
                break
            k, x0, y0 = s
            tries[w, r, 0] = k
            sx, sy = np.append(sx, x0), np.append(sy, y0)
            g = _first_accept(seed, a, 4, side, mr, lambda x, y: _far(x, y, np.float32([x0]), np.float32([y0]), tr2)
                              & _far(x, y, gx, gy, sep2))
            if g is None:
                status[w] = 1 + r
                break
            tries[w, r, 1] = g[0]
            gx, gy = np.append(gx, g[1]), np.append(gy, g[2])
        if status[w]:
            continue
        for r in range(R):
            i = w * R + r
            th = normalize(rand4(seed, (agent0 + r) & 0xFFFFFFFF, 0, [0], 5)[0, 0] * TWO_PI_F)
            pose[i, 0:3] = sx[r], sy[r], th
            goal[i, 0:2] = gx[r], gy[r]
            if cfg.pre_distance_zero:
                pose[i, 3] = 0.0
            else:
                ddx, ddy = _F(gx[r] - sx[r]), _F(gy[r] - sy[r])
                pose[i, 3] = np.sqrt(fmaf(ddx, ddx, _F(ddy * ddy)))
            acc[i, 2:4] = sx[r], sy[r]
    return pose, goal, acc, status, tries
