"""Numpy / float64 restatement of the action sampler rlca_policy_sample (include/rlca.h), written from the rule, not
the kernel.

Row i of a call with (seed, counter) draws Philox-4x32-10 (layout_ref.philox) of the counter
(i, counter lo, counter hi, 0x5A17) under the key (seed lo, seed hi).  The first two output words give the uniforms
u1 = ((w0 >> 8) + 1) 2^-24 in (0, 1] and u2 = (w1 >> 8) 2^-24 in [0, 1), both exact in float32.  The angle is the
float32 product float32(2 pi) * u2, rounded once, as the kernel forms it; everything after it is float64:
z = sqrt(-2 ln u1) (cos t, sin t), action = mean + exp(logstd) z, the log-probability is model/utils.py's
log_normal_density summed over both dimensions, and the scaled action is the action clipped to [[0, -1], [1, 1]]."""
import math

import numpy as np

from layout_ref import TWO_PI_F, philox

PURPOSE = 0x5A17                            # the sampler's Philox purpose word (rlca_env 1-2, rlca_layout 3-5)
BOUND_LO = np.array([0.0, -1.0], np.float32)  # action bound [[v_min, w_min], [v_max, w_max]] (ppo_stage1.py:170)
BOUND_HI = np.array([1.0, 1.0], np.float32)
LOG_SQRT_2PI = 0.5 * math.log(2 * math.pi)
_M32 = 0xFFFFFFFF


def words(seed, counter, nb):
    """(w0, w1) uint64 arrays (nb,): the first two Philox words of rows 0 .. nb-1"""
    seed, counter = int(seed), int(counter)
    n = np.arange(nb, dtype=np.uint64)
    full = lambda v: np.full(nb, v, np.uint64)
    w = philox((n, full(counter & _M32), full(counter >> 32), full(PURPOSE)), seed & _M32, seed >> 32)
    return w[0], w[1]


def uniforms(w0, w1):
    """u1 in (0, 1] and u2 in [0, 1) as float32 (exact): the top 24 bits of each word times 2^-24, u1 moved up by one
    step"""
    w0, w1 = np.asarray(w0, np.uint64), np.asarray(w1, np.uint64)
    u1 = ((w0 >> np.uint64(8)) + np.uint64(1)).astype(np.float64) * 2.0 ** -24
    u2 = (w1 >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    return u1.astype(np.float32), u2.astype(np.float32)


def angle(u2):
    """the float32 product float32(2 pi) * u2, one rounding"""
    return (TWO_PI_F * np.asarray(u2, np.float32)).astype(np.float32)


def box_muller(u1, u2):
    """(z0, z1) float64: sqrt(-2 ln u1) (cos t, sin t) at the float32 angle t"""
    r = np.sqrt(-2.0 * np.log(np.asarray(u1, np.float64)))
    t = angle(u2).astype(np.float64)
    return r * np.cos(t), r * np.sin(t)


def normals(seed, counter, nb):
    """(nb, 2) float64 standard normals of a call"""
    z0, z1 = box_muller(*uniforms(*words(seed, counter, nb)))
    return np.stack([z0, z1], 1)


def sigma(logstd):
    return np.exp(np.asarray(logstd, np.float32).astype(np.float64))


def sample(mean, logstd, seed, counter):
    """float64 action (nb, 2) of mode 0 and the normals z it was drawn from"""
    mean = np.asarray(mean, np.float32).astype(np.float64)
    z = normals(seed, counter, mean.shape[0])
    return mean + sigma(logstd) * z, z


def log_prob(action, mean, logstd):
    """log_normal_density (model/utils.py:90-97) summed over the 2 dimensions, float64, of float32 inputs"""
    a, m = (np.asarray(x, np.float32).astype(np.float64) for x in (action, mean))
    ls = np.asarray(logstd, np.float32).astype(np.float64)
    return (-(a - m) ** 2 / (2 * np.exp(2 * ls)) - LOG_SQRT_2PI - ls).sum(-1)


def scaled(action):
    """the float32 action clipped to the action bound"""
    return np.minimum(np.maximum(np.asarray(action, np.float32), BOUND_LO), BOUND_HI)
