"""Numpy restatement of the acceleration-limit rule (include/rlca.h, DESIGN.md §9r), written from the rule, not the
kernel, in float32 throughout.

Limits: an agent starting an episode draws a = lin_lo + (lin_hi - lin_lo) u0 and b = ang_lo + (ang_hi - ang_lo) u1,
u = (w >> 8) 2^-24 of the first two Philox-4x32-10 words (layout_ref.philox) of (global agent, draw, 0, 0xE6 | stream
<< 8) under the key (seed lo, seed hi), global agent = (world_offset + w) R + r.

Per component: the target is the command with NaN and |x| > 3e38 made 0, clipped to the action bounds; prev is the
value executed on the last call, or 0 for a fresh or crashed row; with d = target - prev and s = limit dt the executed
value is prev + s if d > s, prev - s if d < -s, else the target.  A kind whose range is (0, 0) executes the target."""
import numpy as np

from layout_ref import philox

PURPOSE = 0xE6
_M32 = 0xFFFFFFFF
_F = np.float32


def limits(seed, agents, draw, linear, angular, stream=0):
    """(N, 2) float32 limits of the global agents `agents` drawn at call `draw`"""
    a = np.asarray(agents, np.uint64)
    full = lambda v: np.full(a.shape, v, np.uint64)
    w = philox((a, full(draw), full(0), full(PURPOSE | (stream << 8))), int(seed) & _M32, int(seed) >> 32)
    out = np.empty((a.shape[0], 2), np.float32)
    for k, (lo, hi) in enumerate((linear, angular)):
        u = (w[k] >> np.uint64(8)).astype(np.float32) * _F(2.0 ** -24)
        out[:, k] = _F(lo) + (_F(hi) - _F(lo)) * u
    return out


def target(x, lo, hi):
    """what the tick executes for the command components x"""
    x = np.where(np.abs(x) <= _F(3.0e38), x, _F(0.0)).astype(np.float32)
    return np.where(x < _F(lo), _F(lo), np.where(x > _F(hi), _F(hi), x)).astype(np.float32)


class Dynamics:
    """The rule for N = R W agents of one env handle; one call per tick."""

    def __init__(self, R, W, linear, angular, seed, bounds, dt, world_offset=0, stream=0):
        self.N = R * W
        self.agents = np.uint64(world_offset * R) + np.arange(self.N, dtype=np.uint64)
        self.linear, self.angular, self.seed, self.stream = tuple(linear), tuple(angular), seed, stream
        self.bounds, self.dt = bounds, _F(dt)                # bounds: (v_min, v_max, w_min, w_max)
        self.calls = 0
        self.limit = np.zeros((self.N, 2), np.float32)
        self.vel = np.zeros((self.N, 2), np.float32)

    def action(self, cmd, flags=None):
        """the executed (N, 2) float32 command for the command `cmd`"""
        t = self.calls
        self.calls += 1
        cmd = np.asarray(cmd, np.float32)
        fresh = np.ones(self.N, bool) if flags is None else np.asarray(flags)[:, 3] != 0
        crashed = np.zeros(self.N, bool) if flags is None else np.asarray(flags)[:, 1] != 0
        drawn = limits(self.seed, self.agents, t, self.linear, self.angular, self.stream)
        self.limit[fresh] = drawn[fresh]
        prev = np.where((fresh | crashed)[:, None], _F(0.0), self.vel).astype(np.float32)
        v0, v1, w0, w1 = self.bounds
        out = np.stack([target(cmd[:, 0], v0, v1), target(cmd[:, 1], w0, w1)], 1)
        for k, on in ((0, self.linear[1] > 0), (1, self.angular[1] > 0)):
            if not on:
                continue
            s = (self.limit[:, k] * self.dt).astype(np.float32)
            d = (out[:, k] - prev[:, k]).astype(np.float32)
            out[:, k] = np.where(d > s, prev[:, k] + s, np.where(d < -s, prev[:, k] - s, out[:, k]))
        self.vel = out.copy()
        return out
