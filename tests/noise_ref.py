"""Numpy / float64 restatement of the noise rule (include/rlca.h, DESIGN.md §9p), written from the rule, not the kernel.

Draws: Philox-4x32-10 (layout_ref.philox) of (global agent, draw, element group, purpose | stream << 8) under the key
(seed lo, seed hi); global agent = (world_offset + w) R + r.  Uniforms are the top 24 bits of a word times 2^-24
(exact in float32).  A normal pair from words (a, b): u1 = ((a >> 8) + 1) 2^-24, u2 = (b >> 8) 2^-24, the angle is the
float32 product float32(2 pi) u2 rounded once, and everything after it is float64: z = sqrt(-2 ln u1) (cos, sin).

Scan: group g holds beams 4g .. 4g + 3; range noise takes z0, z1 from words (0, 1) and z2, z3 from words (2, 3) of
purpose 0xE1, dropout the four uniforms of purpose 0xE2.  A dropped beam (u < p) reads range_max; otherwise a beam with
a return (r = (o + 0.5) range_max < range_max) reads clamp(r + sigma z, 0, range_max), normalised r / 6 - 0.5.
Action: z1, z2 from words (0, 1) of purpose 0xE3, group 0; clip, times max(1 + sigma z, 0), clip."""
import numpy as np

from layout_ref import TWO_PI_F, philox

PURPOSE_RANGE, PURPOSE_DROPOUT, PURPOSE_ACTION = 0xE1, 0xE2, 0xE3
U = 2.0 ** -24                    # unit roundoff of float32: half an ulp of 1
_M32 = 0xFFFFFFFF


def words(seed, agents, draw, groups, purpose, stream=0):
    """The four Philox words (uint64 arrays) of the counters (agents, draw, groups, purpose | stream << 8)."""
    agents, groups = np.broadcast_arrays(np.asarray(agents, np.uint64), np.asarray(groups, np.uint64))
    full = lambda v: np.full(agents.shape, v, np.uint64)
    return philox((agents, full(draw), groups, full(purpose | (stream << 8))), int(seed) & _M32, int(seed) >> 32)


def uniform(w):
    """float64 value of the float32 uniform of a word: exact"""
    return (np.asarray(w, np.uint64) >> np.uint64(8)).astype(np.float64) * U


def normal_pair(a, b):
    """(z0, z1, rho) float64 from the words (a, b)"""
    u1 = ((np.asarray(a, np.uint64) >> np.uint64(8)) + np.uint64(1)).astype(np.float64) * U
    u2 = uniform(b).astype(np.float32)
    t = (TWO_PI_F * u2).astype(np.float32).astype(np.float64)
    rho = np.sqrt(-2.0 * np.log(u1))
    return rho * np.cos(t), rho * np.sin(t), rho


def agents(R, W, world_offset=0):
    return (np.uint64(world_offset * R) + np.arange(R * W, dtype=np.uint64))


def scan_draws(seed, R, W, B, draw, world_offset=0, stream=0):
    """(z, rho, u) float64 arrays (N, B): the normal, its radius and the dropout uniform of every beam"""
    G = (B + 3) // 4
    a = np.repeat(agents(R, W, world_offset), G)
    g = np.tile(np.arange(G, dtype=np.uint64), R * W)
    w = words(seed, a, draw, g, PURPOSE_RANGE, stream)
    z0, z1, r01 = normal_pair(w[0], w[1])
    z2, z3, r23 = normal_pair(w[2], w[3])
    z = np.stack([z0, z1, z2, z3], 1).reshape(R * W, 4 * G)[:, :B]
    rho = np.stack([r01, r01, r23, r23], 1).reshape(R * W, 4 * G)[:, :B]
    d = words(seed, a, draw, g, PURPOSE_DROPOUT, stream)
    u = np.stack([uniform(x) for x in d], 1).reshape(R * W, 4 * G)[:, :B]
    return z, rho, u


def scan(newest, params, R, W, draw, range_max=6.0, world_offset=0, stream=0):
    """float64 (N, B) perturbed newest frame from the float32 newest frame (N, B), plus the dropped mask, the normals
    and their radii.  params: dict of range_sigma, dropout, seed."""
    o = np.asarray(newest, np.float32).astype(np.float64)
    N, B = o.shape
    z, rho, u = scan_draws(params['seed'], R, W, B, draw, world_offset, stream)
    p = float(np.float32(params['dropout']))
    sigma = float(np.float32(params['range_sigma']))
    dropped = u < p
    r = (o + 0.5) * range_max
    ret = r < range_max
    rp = np.clip(r + sigma * z, 0.0, range_max)
    out = np.where(ret & (sigma > 0), rp / 6.0 - 0.5, o)
    out = np.where(dropped, range_max / 6.0 - 0.5, out)
    return out, dropped, z, rho


def scan_tolerance(sigma, rho, range_max=6.0):
    """Bound on |kernel - scan()| for a perturbed beam: r recovered from o in float32 (two roundings, < 2^-21 m), the
    normal to 16 U rho (the contract ln within 2 ulps, sqrt, the contract sin / cos and the product, each a few U), the
    fma rounding r + sigma z (half an ulp of 6 m), the float32 1/6 (r' |1/6f - 1/6| < 3.1e-8) and the final rounding
    (half an ulp of 0.5)."""
    return (2.0 ** -21 + sigma * 16 * U * rho + 2.0 ** -22) / 6.0 + range_max * abs(float(np.float32(1 / 6)) - 1 / 6) \
        + 2.0 ** -25


def action_draws(seed, R, W, draw, world_offset=0, stream=0):
    """(z1, z2, rho) float64 (N,) of every agent"""
    w = words(seed, agents(R, W, world_offset), draw, 0, PURPOSE_ACTION, stream)
    return normal_pair(w[0], w[1])


def action(cmd, params, bounds, R, W, draw, world_offset=0, stream=0):
    """float64 (N, 2) executed command, the normals and their radius.  bounds: (v_min, v_max, w_min, w_max)."""
    c = np.asarray(cmd, np.float32).astype(np.float64)
    lo = np.array([bounds[0], bounds[2]], np.float64)
    hi = np.array([bounds[1], bounds[3]], np.float64)
    c = np.minimum(np.maximum(c, lo), hi)
    z1, z2, rho = action_draws(params['seed'], R, W, draw, world_offset, stream)
    s = np.array([float(np.float32(params['v_gain_sigma'])), float(np.float32(params['w_gain_sigma']))])
    g = np.maximum(1.0 + s * np.stack([z1, z2], 1), 0.0)
    return np.minimum(np.maximum(c * g, lo), hi), np.stack([z1, z2], 1), rho


def action_tolerance(cmd, sigma, rho):
    """Bound on |kernel - action()|: the normal to 16 U rho, the gain's fma (half an ulp of the gain), the product
    (half an ulp of the result)."""
    c = np.abs(np.asarray(cmd, np.float64))
    g = 1.0 + sigma * rho
    return c * (sigma * 16 * U * rho + 2 * U * g) + 2 * U * c * g
