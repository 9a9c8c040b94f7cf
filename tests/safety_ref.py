"""Numpy restatement of the safety metrics (DESIGN.md §9m), written from the definitions, not from csrc/rlca_safety.cu:
footprint corners by the §4 corner formula (sincos polynomial and exactly rounded fmaf), separation (separating-axis
test, then the 32 corner-to-edge distances), clearance, the contact bound, the per-episode fold and the float64
reduction.  float32 arithmetic, one rounding per operation."""
import numpy as np

_F = np.float32
INF = _F(np.inf)
COLUMNS = ('crash_static', 'crash_robot', 'crash_both_in_range', 'crash_into_masked', 'reached', 'reached_separation',
           'sum_separation', 'sum_separation_sq', 'reached_clearance', 'sum_clearance', 'sum_clearance_sq',
           'near_episodes', 'sum_near_ticks', 'min_separation')


def fmaf(a, b, c):
    """round_f32(a * b + c) with one rounding: the float64 product is exact, the float64 sum's error is recovered
    (TwoSum) and decides the float32 rounding where the float64 sum sits exactly between two float32 values."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    up, dn = np.nextafter(r, INF), np.nextafter(r, -INF)
    d = s - r64
    r = np.where((d == (up.astype(np.float64) - r64) / 2) & (e > 0), up, r)
    r = np.where((-d == (r64 - dn.astype(np.float64)) / 2) & (e < 0), dn, r)
    return r.astype(np.float32)


def sincos(x):
    """sin, cos of the numerics contract (DESIGN.md §4)."""
    x = np.asarray(x, np.float32)
    q = np.rint(x * _F(0.636619772367581343)).astype(np.float32)
    r = fmaf(q, _F(-1.57079625129699707031), x)
    r = fmaf(q, _F(-7.54978941586159635335e-08), r)
    r2 = r * r
    ps = fmaf(r2, _F(-1.9515295891e-4), _F(8.3321608736e-3))
    ps = fmaf(r2, ps, _F(-1.6666654611e-1))
    sr = fmaf(r * r2, ps, r)
    pc = fmaf(r2, _F(2.443315711809948e-5), _F(-1.388731625493765e-3))
    pc = fmaf(r2, pc, _F(4.166664568298827e-2))
    cr = fmaf(r2 * r2, pc, fmaf(r2, _F(-0.5), _F(1.0)))
    qi = q.astype(np.int64) & 3
    s = np.where(qi & 1, cr, sr)
    c = np.where(qi & 1, sr, cr)
    s = np.where(qi >= 2, -s, s)
    c = np.where((qi == 1) | (qi == 2), -c, c)
    return s.astype(np.float32), c.astype(np.float32)


def corners(pose, half_len, half_wid):
    """(n, 4, 2) footprint corners of pose (n, >= 3), counter-clockwise from (-half_len, -half_wid)."""
    pose = np.asarray(pose, np.float32)
    x, y = pose[:, 0], pose[:, 1]
    s, c = sincos(pose[:, 2])
    hl, hw = _F(half_len), _F(half_wid)
    out = np.zeros((len(pose), 4, 2), np.float32)
    for k, (hx, hy) in enumerate(((-hl, -hw), (hl, -hw), (hl, hw), (-hl, hw))):
        out[:, k, 0] = fmaf(hx, c, fmaf(-hy, s, x))
        out[:, k, 1] = fmaf(hx, s, fmaf(hy, c, y))
    return out


def _axis_separates(P, k, A, B):
    dx = (P[:, k + 1, 0] - P[:, k, 0])[:, None]
    dy = (P[:, k + 1, 1] - P[:, k, 1])[:, None]
    pa = A[:, :, 0] * dx + A[:, :, 1] * dy
    pb = B[:, :, 0] * dx + B[:, :, 1] * dy
    return (pa.max(1) < pb.min(1)) | (pb.max(1) < pa.min(1))


def _point_segment_sq(p, a, b):
    ex, ey = b[:, 0] - a[:, 0], b[:, 1] - a[:, 1]
    wx, wy = p[:, 0] - a[:, 0], p[:, 1] - a[:, 1]
    t = (wx * ex + wy * ey) / (ex * ex + ey * ey)
    t = np.minimum(np.maximum(t, _F(0.0)), _F(1.0))
    dx, dy = wx - t * ex, wy - t * ey
    return dx * dx + dy * dy


def separation(A, B):
    """(n,) distance between the rectangles A[i] and B[i] ((n, 4, 2) corners): 0 when no edge direction of either
    separates them, else the square root of the least squared corner-to-edge distance."""
    A, B = np.asarray(A, np.float32), np.asarray(B, np.float32)
    apart = _axis_separates(A, 0, A, B) | _axis_separates(A, 1, A, B) | _axis_separates(B, 0, A, B) | \
        _axis_separates(B, 1, A, B)
    m = np.full(len(A), INF, np.float32)
    for P, Q in ((A, B), (B, A)):
        for i in range(4):
            for k in range(4):
                m = np.minimum(m, _point_segment_sq(P[:, i], Q[:, k], Q[:, (k + 1) & 3]))
    return np.where(apart, np.sqrt(m), _F(0.0)).astype(np.float32)


def contact(cfg):
    """sqrt(2) resolution + 2 dt (v_max + max(|w_min|, |w_max|) r_c), left to right in float32."""
    hl, hw = _F(cfg.half_len), _F(cfg.half_wid)
    r_c = np.sqrt(hl * hl + hw * hw)
    w_abs = max(abs(_F(cfg.w_min)), abs(_F(cfg.w_max)))
    return _F(_F(1.41421356) * _F(cfg.resolution) + _F(2.0) * _F(cfg.dt) * (_F(cfg.v_max) + w_abs * r_c))


def clearance(obs, range_max):
    return ((np.asarray(obs, np.float32).min(1) + _F(0.5)) * _F(range_max)).astype(np.float32)


def world_separations(C, R):
    """(W, R, R) separation of every ordered pair of each world from corners C (W * R, 4, 2); +inf on the diagonal."""
    W = len(C) // R
    a, b = np.meshgrid(np.arange(R), np.arange(R), indexing='ij')
    S = np.full((W, R, R), INF, np.float32)
    up = a < b
    for w in range(W):
        Cw = C[w * R:(w + 1) * R]
        s = separation(Cw[a[up]], Cw[b[up]])
        S[w][a[up], b[up]] = s
        S[w][b[up], a[up]] = s
    return S


class Tracker:
    """The episode tracker's boundaries (closed, count) and the safety fold next to them."""

    def __init__(self, cfg, episodes, near_dist):
        self.cfg, self.E, self.near_dist = cfg, int(episodes), _F(near_dist)
        N = cfg.robots_per_world * cfg.num_worlds
        self.closed = np.full(N, -1, np.int32)
        self.count = np.zeros(N, np.int32)
        self.min_sep = np.full(N, INF, np.float32)
        self.min_clear = np.full(N, INF, np.float32)
        self.last_clear = np.full(N, INF, np.float32)
        self.near = np.zeros(N, np.int32)
        self.partner = np.full(N, -1, np.int32)
        self.records = np.zeros((N, self.E, 4), np.float32)
        self.results = np.zeros((N, self.E, 4), np.float32)        # the tracker's records: result code in [..., 0]

    def state(self):
        return {k: getattr(self, k) for k in ('min_sep', 'min_clear', 'last_clear', 'near', 'partner', 'records')}

    def tick(self, pose_in, meta_in, pose_out, flags, obs):
        cfg, R = self.cfg, self.cfg.robots_per_world
        S_in = world_separations(corners(pose_in, cfg.half_len, cfg.half_wid), R)
        S_out = world_separations(corners(pose_out, cfg.half_len, cfg.half_wid), R)
        clear = clearance(obs, cfg.range_max)
        bound = contact(cfg)
        for a in range(len(pose_in)):
            w, r = divmod(a, R)
            done, crashed, result, respawned = (int(v) for v in flags[a])
            ep = int(meta_in[a][1])
            if self.closed[a] != ep:
                row = S_in[w, r] if respawned else S_out[w, r]
                j = int(np.argmin(row))                               # the lowest index on ties
                s = row[j]
                if s < self.min_sep[a]:
                    self.min_sep[a], self.partner[a] = s, j
                if not respawned:
                    self.min_clear[a] = min(self.min_clear[a], clear[a])
                self.near[a] += int(s < self.near_dist)
                if result != 0:
                    c = int(self.count[a])
                    if c < self.E:
                        cause, hit = 0, -1
                        if result == 2:
                            j0 = int(np.argmin(S_in[w, r]))
                            if S_in[w, r, j0] > bound:
                                cause = 1
                            else:
                                cause, hit = 2 | (4 if self.last_clear[a] < bound else 0), j0
                        packed = cause | (hit + 1) << 8 | (int(self.partner[a]) + 1) << 16
                        self.records[a, c] = (self.min_sep[a], self.min_clear[a], self.near[a], packed)
                        self.results[a, c, 0] = result
                    self.count[a] = c + 1
                    self.closed[a] = ep
                    respawned = 1
            if respawned:
                self.min_sep[a], self.min_clear[a], self.near[a], self.partner[a] = INF, INF, 0, -1
            self.last_clear[a] = clear[a]


def reduce(R, records, results, count, mask=None, split=False, want=0, world=0):
    """The partials of one world, float64, agents then records; `results[..., 0]` is the tracker's result code."""
    s = dict.fromkeys(COLUMNS, np.float64(0.0))
    s['min_separation'] = np.float64(np.inf)
    E = records.shape[1]
    for r in range(R):
        a = world * R + r
        if split and (mask[a] != 0) != bool(want):
            continue
        for i in range(min(int(count[a]), E)):
            sep, clr, near, packed = records[a, i]
            sep, clr, near, packed = np.float64(sep), np.float64(clr), np.float64(near), int(packed)
            s['min_separation'] = min(s['min_separation'], sep)
            cause, hit = packed & 3, ((packed >> 8) & 0xff) - 1
            if cause == 1:
                s['crash_static'] += 1.0
            if cause == 2:
                s['crash_robot'] += 1.0
                if packed & 4:
                    s['crash_both_in_range'] += 1.0
                if mask is not None and hit >= 0 and mask[world * R + hit]:
                    s['crash_into_masked'] += 1.0
            if int(results[a, i, 0]) != 1:
                continue
            s['reached'] += 1.0
            if np.isfinite(sep):
                s['reached_separation'] += 1.0
                s['sum_separation'] += sep
                s['sum_separation_sq'] += sep * sep
            if np.isfinite(clr):
                s['reached_clearance'] += 1.0
                s['sum_clearance'] += clr
                s['sum_clearance_sq'] += clr * clr
            if near > 0:
                s['near_episodes'] += 1.0
            s['sum_near_ticks'] += near
    return np.array([s[k] for k in COLUMNS], np.float64)
