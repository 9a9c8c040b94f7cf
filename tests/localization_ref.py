"""Numpy restatement of the localization-error rule (include/rlca.h, DESIGN.md §9s), written from the rule, not the
kernel, in float32 throughout with one rounding per operation: the contract sin / cos of DESIGN.md §4 (safety_ref) and
the contract ln (cephes logf on the mantissa, explicit FMAs) restated here.

Draws: Philox-4x32-10 (layout_ref.philox) of (global agent, draw, group, 0xE7 | stream << 8) under the key (seed lo,
seed hi).  Group 0: normals of ex, ey from words (0, 1) and of etheta, v from words (2, 3); group 1: the normal of w
from words (0, 1) and the uniforms of sigma_xy (word 2) and sigma_theta (word 3).  A normal pair from words (a, b):
u1 = ((a >> 8) + 1) 2^-24, u2 = (b >> 8) 2^-24, rho = sqrt(-2 ln u1), (rho cos t, rho sin t) with t = 2 pi u2.

Error, per component: a fresh row (every row without flags, else was_reset) draws sigma = lo + (hi - lo) u and takes
e = sigma xi; any other row e = rho e + kappa (sigma xi), or e itself when kappa = 0.  rho = exp(-dt / tau) and kappa =
sqrt(1 - rho^2) in float64, rounded to float32.  Believed pose: x + ex, y + ey, theta + etheta, each only when its error
is not 0; the local goal is ((gx - x') c + (gy - y') s, (gy - y') c - (gx - x') s) with (s, c) = sincos(theta'), each
component one FMA over a rounded product; v and w are gs's plus sigma z when sigma > 0."""
import math

import numpy as np

from layout_ref import philox
from safety_ref import fmaf, sincos

PURPOSE = 0xE7
_F = np.float32
_M32 = 0xFFFFFFFF
_U = _F(2.0 ** -24)


def logf(x):
    """ln of positive normal float32 x under the numerics contract"""
    x = np.asarray(x, np.float32)
    b = x.view(np.uint32).astype(np.int64)
    e = (b >> 23) - 127
    m = ((b & 0x007FFFFF) | 0x3F800000).astype(np.uint32).view(np.float32)
    big = m > _F(1.41421356237309505)
    m = np.where(big, m * _F(0.5), m).astype(np.float32)
    e = np.where(big, e + 1, e)
    f = (m - _F(1.0)).astype(np.float32)
    z = (f * f).astype(np.float32)
    fe = e.astype(np.float32)
    p = fmaf(_F(7.0376836292e-2), f, _F(-1.1514610310e-1))
    for c in (1.1676998740e-1, -1.2420140846e-1, 1.4249322787e-1, -1.6668057665e-1, 2.0000714765e-1,
              -2.4999993993e-1, 3.3333331174e-1):
        p = fmaf(p, f, _F(c))
    y = fmaf((p * f).astype(np.float32), z, (fe * _F(-2.12194440e-4)).astype(np.float32))
    y = fmaf(_F(-0.5), z, y)
    return fmaf(fe, _F(0.693359375), (f + y).astype(np.float32))


def normal_pair(a, b):
    """float32 Box-Muller pair of the words (a, b) (uint64 arrays)"""
    u1 = ((np.asarray(a, np.uint64) >> np.uint64(8)).astype(np.float32) + _F(1.0)) * _U
    u2 = (np.asarray(b, np.uint64) >> np.uint64(8)).astype(np.float32) * _U
    rho = np.sqrt((_F(-2.0) * logf(u1)).astype(np.float32))
    s, c = sincos((_F(6.28318548202514648438) * u2).astype(np.float32))
    return (rho * c).astype(np.float32), (rho * s).astype(np.float32)


def uniform(w):
    return (np.asarray(w, np.uint64) >> np.uint64(8)).astype(np.float32) * _U


def coefficients(tau, dt):
    """(rho, kappa) float32 of the correlation time tau s at the tick dt s"""
    tau, dt = float(np.float32(tau)), float(np.float32(dt))
    if tau == 0.0:
        return _F(0.0), _F(1.0)
    if math.isinf(tau):
        return _F(1.0), _F(0.0)
    rho = math.exp(-dt / tau)
    return _F(rho), _F(math.sqrt(1.0 - rho * rho))


def goal_speed(pose, goal, s, c):
    """(N, 2) local goal of the poses (N, >= 2) with heading sin / cos s, c"""
    ddx = (goal[:, 0] - pose[:, 0]).astype(np.float32)
    ddy = (goal[:, 1] - pose[:, 1]).astype(np.float32)
    return np.stack([fmaf(ddx, c, (ddy * s).astype(np.float32)), fmaf(ddy, c, -(ddx * s).astype(np.float32))], 1)


class Localization:
    """The rule for N = R W agents of one env handle; one call per tick."""

    def __init__(self, R, W, pose_sigma, heading_sigma, tau, speed_sigma, seed, dt, world_offset=0, stream=0):
        self.N = R * W
        self.agents = np.uint64(world_offset * R) + np.arange(self.N, dtype=np.uint64)
        self.pose_sigma = tuple(_F(v) for v in pose_sigma)
        self.heading_sigma = tuple(_F(v) for v in heading_sigma)
        self.speed_sigma = tuple(_F(v) for v in speed_sigma)
        self.rho, self.kappa = coefficients(tau, dt)
        self.seed, self.stream = int(seed), stream
        self.calls = 0
        self.err = np.zeros((self.N, 3), np.float32)
        self.sigma = np.zeros((self.N, 2), np.float32)

    def _words(self, group):
        full = lambda v: np.full(self.N, v, np.uint64)
        return philox((self.agents, full(self.calls), full(group), full(PURPOSE | (self.stream << 8))),
                      self.seed & _M32, self.seed >> 32)

    def observe(self, pose, goal, gs, flags=None):
        """the believed (N, 4) float32 gs"""
        pose, goal, gs = (np.asarray(a, np.float32) for a in (pose, goal, gs))
        w0, w1 = self._words(0), self._words(1)
        self.calls += 1
        zx, zy = normal_pair(w0[0], w0[1])
        zt, zv = normal_pair(w0[2], w0[3])
        zw, _ = normal_pair(w1[0], w1[1])
        fresh = np.ones(self.N, bool) if flags is None else np.asarray(flags)[:, 3] != 0
        for k, (lo, hi), w in ((0, self.pose_sigma, w1[2]), (1, self.heading_sigma, w1[3])):
            drawn = (lo + ((hi - lo).astype(np.float32) * uniform(w)).astype(np.float32)).astype(np.float32)
            self.sigma[fresh, k] = drawn[fresh]
        for k, (z, sg) in enumerate(((zx, self.sigma[:, 0]), (zy, self.sigma[:, 0]), (zt, self.sigma[:, 1]))):
            n = (sg * z).astype(np.float32)
            if self.kappa == 0.0:
                step = self.err[:, k]
            else:
                step = ((self.rho * self.err[:, k]).astype(np.float32) + (self.kappa * n).astype(np.float32))
            self.err[:, k] = np.where(fresh, n, step.astype(np.float32))
        believed = pose[:, 0:3].copy()
        for k in range(3):
            believed[:, k] = np.where(self.err[:, k] != 0, (pose[:, k] + self.err[:, k]).astype(np.float32),
                                      pose[:, k])
        s, c = sincos(believed[:, 2])
        out = np.empty((self.N, 4), np.float32)
        out[:, 0:2] = goal_speed(believed, goal, s, c)
        for k, (sv, z) in enumerate(((self.speed_sigma[0], zv), (self.speed_sigma[1], zw))):
            out[:, 2 + k] = (gs[:, 2 + k] + (sv * z).astype(np.float32)).astype(np.float32) if sv > 0 else gs[:, 2 + k]
        return out
