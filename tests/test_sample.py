"""The action sampler's reference without a GPU: Philox-4x32-10 against the published known answers, the float64
restatement in sample_ref.py against closed forms and scipy, and the arguments rlca_policy_sample rejects before it
launches anything."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy import stats

import sample_ref as ref
from layout_ref import philox

RLCA_ERR_INVALID = 1

# Random123's kat_vectors for philox4x32_10: counter (4 words), key (2 words) -> output (4 words)
PHILOX_KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
     (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff),
     (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize('kat', range(len(PHILOX_KAT)))
def test_philox_known_answers(kat):
    """layout_ref.philox is the published Philox-4x32-10.  The GPU layout and env tests hold the device generator
    (dev_philox, which the env, the layouts and the action sampler share) bit for bit to layout_ref, so this pins all of
    them to the algorithm, not just to each other."""
    ctr, key, want = PHILOX_KAT[kat]
    got = philox([np.array([c], np.uint64) for c in ctr], *key)
    assert [int(w[0]) for w in got] == list(want), [hex(int(w[0])) for w in got]


def test_counter_and_key_layout():
    """row i of (seed, counter) is Philox of (i, counter lo, counter hi, 0x5A17) under (seed lo, seed hi)"""
    seed, counter = 0x0123456789ABCDEF, 0xFEDCBA9876543210
    w0, w1 = ref.words(seed, counter, 5)
    for i in range(5):
        out = philox([np.array([v], np.uint64) for v in (i, 0x76543210, 0xFEDCBA98, 0x5A17)], 0x89ABCDEF, 0x01234567)
        assert (int(w0[i]), int(w1[i])) == (int(out[0][0]), int(out[1][0]))


def test_uniform_ends():
    """u1 = ((w0 >> 8) + 1) 2^-24 covers (0, 1], u2 = (w1 >> 8) 2^-24 covers [0, 1), exactly in float32"""
    w = np.array([0, 0xFF, 0x100, 0x7FFFFFFF, 0xFFFFFF00, 0xFFFFFFFF], np.uint64)
    u1, u2 = ref.uniforms(w, w)
    assert u1.dtype == np.float32 and u2.dtype == np.float32
    assert u1.tolist() == [2.0 ** -24, 2.0 ** -24, 2.0 ** -23, 0.5, 1.0, 1.0]
    assert u2.tolist() == [0.0, 0.0, 2.0 ** -24, 0.5 - 2.0 ** -24, 1.0 - 2.0 ** -24, 1.0 - 2.0 ** -24]


def test_box_muller_radius_ends_and_angle_rounding():
    """u1 = 1 gives r = 0; the smallest u1, 2^-24, gives the largest radius sqrt(48 ln 2) ~ 5.77; the angle is the
    float32 product of float32(2 pi) and u2, not the exact 2 pi u2"""
    z0, z1 = ref.box_muller(np.float32([1.0, 1.0]), np.float32([0.0, 0.3]))
    assert z0.tolist() == [0.0, 0.0] and z1.tolist() == [0.0, 0.0]
    u2 = np.float32([0.0, 0.125, 0.25, 0.5, 0.75, 1 - 2.0 ** -24, 0.1234567])
    z0, z1 = ref.box_muller(np.full(u2.shape, 2.0 ** -24, np.float32), u2)
    r = np.hypot(z0, z1)
    assert np.allclose(r, math.sqrt(48 * math.log(2)), rtol=1e-15, atol=0)
    t = ref.angle(u2)
    assert t.dtype == np.float32
    assert np.array_equal(t, np.float32(6.28318548202514648438) * u2)
    assert np.allclose(np.arctan2(z1, z0) % (2 * np.pi), t.astype(np.float64) % (2 * np.pi), rtol=0, atol=1e-14)
    # the float32 angle differs from 2 pi u2 by up to half an ulp of 2 pi: ~1.7e-7 rad, 1e-6 at r = 5.8
    exact = 2 * np.pi * u2.astype(np.float64)
    assert 0 < np.abs(t - exact).max() <= 2.0 ** -22


def test_log_prob_is_scipy_normal_logpdf():
    rs = np.random.RandomState(3)
    for ls in ([-5.0, 2.0], [-1.85, -1.04], [0.0, 0.0]):
        ls = np.float32(ls)
        mean = np.stack([rs.uniform(0, 1, 1000), rs.uniform(-1, 1, 1000)], 1).astype(np.float32)
        act = (mean + ref.sigma(ls) * rs.uniform(-40, 40, (1000, 2))).astype(np.float32)
        want = stats.norm.logpdf(act.astype(np.float64), mean.astype(np.float64), ref.sigma(ls)).sum(1)
        got = ref.log_prob(act, mean, ls)
        assert np.allclose(got, want, rtol=1e-13, atol=1e-13), np.abs(got - want).max()


def test_sample_is_mean_plus_sigma_z():
    mean = np.float32([[0.25, -0.5], [0.75, 0.5], [0.5, 0.0]])
    ls = np.float32([-1.85, -1.04])
    a, z = ref.sample(mean, ls, 7, 11)
    assert np.array_equal(z, ref.normals(7, 11, 3))
    assert np.array_equal(a, mean.astype(np.float64) + np.exp(ls.astype(np.float64)) * z)
    assert np.abs(z).max() <= math.sqrt(48 * math.log(2))


def test_scaled_clip():
    a = np.float32([[-0.5, -2.0], [0.0, -1.0], [1.0, 1.0], [2.0, 3.0], [0.5, 0.25], [-np.inf, np.inf]])
    assert ref.scaled(a).tolist() == [[0.0, -1.0], [0.0, -1.0], [1.0, 1.0], [1.0, 1.0], [0.5, 0.25], [0.0, 1.0]]


def test_sample_rejects_bad_arguments(built):
    """Each rejected call returns RLCA_ERR_INVALID before anything is launched: on a machine without a GPU an accepted
    call would fail at the launch with a CUDA error instead."""
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    have_gpu = torch.cuda.is_available()
    if have_gpu:      # real buffers: the accepted control call below draws into them
        bufs = [torch.zeros(64, device='cuda') for _ in range(5)]
        params, mean, action, logprob, scaled = (b.data_ptr() for b in bufs)
    else:             # never dereferenced: every call but the control returns before the launch
        params, mean, action, logprob, scaled = (0x10000 * (k + 1) for k in range(5))

    def call(nb=4, mode=0, **null):
        p = dict(params=params, mean=mean, action=action, logprob=logprob)
        p.update({k: 0 for k in null})
        return lib.rlca_policy_sample(C.c_void_p(p['params']), C.c_void_p(p['mean']), nb, 1, 1, mode,
                                      C.c_void_p(p['action']), C.c_void_p(p['logprob']), C.c_void_p(scaled), None)

    bad = {'deterministic -1': dict(mode=-1), 'deterministic 3': dict(mode=3), 'deterministic 2^31 - 1':
           dict(mode=2 ** 31 - 1), 'deterministic -2^31': dict(mode=-2 ** 31), 'nb 0': dict(nb=0),
           'nb -1': dict(nb=-1), 'NULL params': dict(params=1), 'NULL mean': dict(mean=1),
           'NULL action': dict(action=1), 'NULL logprob': dict(logprob=1)}
    for what, kw in bad.items():
        for mode in ((kw.pop('mode'),) if 'mode' in kw else (0, 1, 2)):
            assert call(mode=mode, **kw) == RLCA_ERR_INVALID, (what, mode)
            assert lib.rlca_last_error(), (what, mode)
    if have_gpu:
        for mode in (0, 1, 2):
            assert call(mode=mode) == 0
        torch.cuda.synchronize()
    else:
        assert call() not in (0, RLCA_ERR_INVALID), 'a valid call on a machine without a GPU must fail at the launch'
