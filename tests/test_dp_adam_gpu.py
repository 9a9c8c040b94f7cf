"""The data-parallel optimizer step (csrc/rlca_dp.cu, rlca_adam_step_allreduce) with G simulated ranks on one GPU.

The kernel's peer path takes plain device pointers, so rank q is a set of four buffers (gradient, parameters, both
Adam moments) on the same device, and the G launches of one step run in rank order on one stream: the order that the
two cross-GPU barriers around the launch give a real run.  Every buffer is n + 64 floats long; the 64-float tail, and
with sharded moments everything of a rank's moments outside its own shard, holds a quiet-NaN sentinel, so a stray read
poisons the result and a stray write shows in the bits.

Each step is checked three ways:
  * bit for bit against rlca_adam_step (the single-GPU kernel) on the float32 sum ((g0 + g1) + g2) + ... of the rank
    gradients, with the same grad_scale and step count: the parameters of every rank, and the moments (replicated on
    every rank, or gathered from the shard owners);
  * against Adam in float64 (torch.optim.Adam semantics, bias corrections in float64) on the float64 gradient sum,
    within a first-order bound of the kernel's float32 rounding derived element by element (adam64_with_bound);
  * the shards: disjoint, covering [0, n), equal to parallel.PeerAdam.shard, nothing written outside them or into a
    tail, and the same bits when the ranks launch in reverse order.

A last test takes Adam.step's peer branch on a real CNNPolicy: the fused kernel with G = 1 on the policy's own buffers
skips rlca_policy_adam_step, so the next forward must re-split the fc1 weights and rebuild the conv image.

Each float64 comparison prints `[ratio] <what>: r` (largest error / bound over the elements); run with -s."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from golden_inputs import synthetic_state_dict
from learner_ref import Checks, check_forward, decisive_pool, params64, ref_forward

pytestmark = pytest.mark.gpu

TAIL = 64
SENTINEL = 0x7FC0DEAD                      # a quiet NaN with a payload
U = 2.0 ** -24                             # unit roundoff of float32
LR, BETA1, BETA2, EPS = 1e-3, 0.9, 0.999, 1e-8
STEPS = (1, 2, 3, 10000)                   # 10000: both bias corrections are 1 to float32 precision
WORLDS = (1, 2, 3, 4, 5, 7, 8, 16)
SIZES = (4, 8, 12, 60, 1028, 'flat')       # 'flat': the policy's flat buffer, 2.17 M floats
SLACK = 1.001                              # covers the second-order terms the bound leaves out


def f32(x):
    return float(np.float32(x))


def lib_and_stream():
    from rl_collision_avoidance_b200 import _lib
    return _lib, _lib.load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)


def flat_size():
    from rl_collision_avoidance_b200.model.net import TENSORS
    _, lib, _ = lib_and_stream()
    return int(lib.rlca_policy_param_offset(len(TENSORS)))


def kernel_shard(n, world, rank):
    chunk = -(-(n // 4) // world) * 4
    lo = min(rank * chunk, n)
    return lo, min(lo + chunk, n)


def peer_shard(n, world, rank):
    from rl_collision_avoidance_b200.parallel import PeerAdam
    pa = PeerAdam.__new__(PeerAdam)           # only the fields shard() reads
    pa.n, pa.world = n, world
    return pa.shard(rank)


def sentinel(n):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device='cuda').view(torch.float32)


def bits(t):
    return t.view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def first_diff(a, b):
    d = (bits(a) != bits(b)).nonzero()
    return f'{int(d.numel())} differ, first at {int(d[0])}' if d.numel() else 'equal'


class Ranks:
    """G simulated ranks: rank q's grad, param, m and v, each n + TAIL floats.  Parameters start equal on every rank;
    the moments start at zero, on every rank (replicated) or on the rank's own shard only (sharded)."""

    KINDS = ('grad', 'param', 'm', 'v')

    def __init__(self, G, n, p0, replicate):
        self.G, self.n, self.replicate = G, n, replicate
        self.buf = {k: [sentinel(n + TAIL) for _ in range(G)] for k in self.KINDS}
        for q in range(G):
            self.buf['param'][q][:n] = p0
            lo, hi = (0, n) if replicate else kernel_shard(n, G, q)
            self.buf['m'][q][lo:hi] = 0
            self.buf['v'][q][lo:hi] = 0
        self.ptrs = [(C.c_uint64 * G)(*[t.data_ptr() for t in self.buf[k]]) for k in self.KINDS]

    def step(self, grads, step, scale, order):
        _lib, lib, st = lib_and_stream()
        for q in range(self.G):
            self.buf['grad'][q][:self.n] = grads[q]
        for q in order:
            _lib.check(lib.rlca_adam_step_allreduce(*self.ptrs, 0, 0, 0, 0, q, self.G, self.n, LR, BETA1, BETA2, EPS, step,
                                                    scale, int(self.replicate), st))

    def moments(self, k):
        """m or v of the whole buffer: rank 0's copy, or every shard from its owner"""
        if self.replicate:
            return self.buf[k][0][:self.n].clone()
        return torch.cat([self.buf[k][q][slice(*kernel_shard(self.n, self.G, q))] for q in range(self.G)])


def rank_grads(G, n, gen):
    """one step's gradients of G ranks: normal values of scale 0.1 and, by element class (index mod 8), exact zeros on
    every rank at every step (v stays 0, so the denominator is eps), zeros on some ranks, tiny values (~1e-8), large
    ones (~1e3), and values of alternating sign across the ranks whose sum cancels"""
    i = torch.arange(n, device='cuda')
    cls = i % 8
    out = []
    shared = torch.randn(n, device='cuda', generator=gen)
    for q in range(G):
        g = torch.randn(n, device='cuda', generator=gen) * 0.1
        g = torch.where(cls == 2, g * 1e-7, g)
        g = torch.where(cls == 3, g * 1e4, g)
        g = torch.where(cls == 4, shared * (1 if q % 2 == 0 else -1) + g * 1e-3, g)
        g = torch.where((cls == 1) & ((i // 8 + q) % 3 == 0), 0.0, g)
        g = torch.where(cls == 0, 0.0, g)
        out.append(g.contiguous())
    return out


def adam64_with_bound(grads, scale, p0, m0, v0, step):
    """One Adam step in float64 (torch.optim.Adam with the kernel's float32 lr, betas, eps and grad_scale, bias
    corrections in float64) on the float64 sum of the rank gradients, and a first-order bound, per element, of the
    error of the float32 kernel, which
      sums the G gradients in float32:         |S~ - S| <= gamma(G - 1) sum_q |g_q|
      scales, then forms m and v with one fma: g~ = fl(S~ s), m~ = fl(b1 m0 + fl((1 - b1) g~)),
                                               v~ = fl(b2 v0 + fl(fl((1 - b2) g~) g~))   (1 - b is exact in float32)
      takes bc = 1 - powf(b, step) on the host in float32: |bc~ - bc| <= ulp(b^step) + u bc (powf within 1 ulp)
      rounds sqrt(v), sqrt(bc2), sqrt(v) / sqrt(bc2), + eps, m / denom, lr / bc1 and p - (lr / bc1)(m / denom) once
      each (the last with or without a contracted fma).
    The bound is tight: one rounding to nearest comes within a hair of u |x| for an x just above a power of two, so
    worst-case ratios close to 1 are expected over two million elements; a ratio above 1 is an error.
    Returns (p, m, v) in float64 and their bounds."""
    G = len(grads)
    lr, b1, b2, eps, s = f32(LR), f32(BETA1), f32(BETA2), f32(EPS), f32(scale)
    c1, c2 = 1.0 - b1, 1.0 - b2
    g64 = [g.double() for g in grads]
    S = sum(g64[1:], g64[0])
    A = sum((x.abs() for x in g64[1:]), g64[0].abs())
    p0, m0, v0 = p0.double(), m0.double(), v0.double()
    g = S * s
    m = b1 * m0 + c1 * g
    v = b2 * v0 + c2 * g * g
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    sv = v.sqrt()
    den = sv / math.sqrt(bc2) + eps
    q = m / den
    c = lr / bc1
    d = c * q
    p = p0 - d
    # the bound, term by term
    gamma = (G - 1) * U / (1 - (G - 1) * U)
    ag = g.abs()
    e_g = s * gamma * A * (1 + U) + U * ag
    e_m = c1 * e_g + U * c1 * ag + U * m.abs()
    e_v = c2 * (2 * ag * e_g + e_g * e_g) + 2 * U * c2 * ag * ag + U * v
    e_sq = torch.where(e_v > 0, torch.minimum(e_v.sqrt(), e_v / sv), torch.zeros_like(e_v)) + U * (sv + e_v.sqrt())
    eps_bc = lambda b, bc: (float(np.spacing(np.float32(b ** step))) + U * bc) / bc
    eps_bs = eps_bc(b2, bc2) / 2 + U                                     # sqrtf of the float32 bc2
    bs = math.sqrt(bc2)
    r = sv / bs
    e_r = e_sq / bs + r * (eps_bs + U)
    e_den = e_r + U * den
    e_q = e_m / den + q.abs() * e_den / den + U * q.abs()
    eps_c = eps_bc(b1, bc1) + U
    e_p = c * e_q + d.abs() * (eps_c + U) + U * p.abs()
    return (p, m, v), (SLACK * e_p, SLACK * e_m, SLACK * e_v)


def ratio(got, ref, bound):
    """largest |got - ref| / bound over the elements (an element with a zero bound must be exact)"""
    err = (got.double() - ref).abs()
    if bool((err[bound == 0] > 0).any()):
        return math.inf
    r = err / torch.where(bound > 0, bound, torch.ones_like(bound))
    return float(r.max()) if r.numel() else 0.0


@pytest.mark.parametrize('n', SIZES, ids=[f'n{s}' for s in SIZES])
@pytest.mark.parametrize('G', WORLDS, ids=[f'G{g}' for g in WORLDS])
def test_adam_step_allreduce_simulated_ranks(built, G, n):
    """G ranks x n floats, sharded and replicated moments, grad_scale 1 / G and 1, steps 1, 2, 3 and 10000"""
    _lib, lib, st = lib_and_stream()
    n = flat_size() if n == 'flat' else n
    check = Checks()
    worst = {}
    for replicate in (0, 1):
        for scale in (1.0 / G, 1.0):
            tag = f'{"replicated" if replicate else "sharded"} scale={scale:.3g}'
            gen = torch.Generator(device='cuda').manual_seed(1000 * G + 10 * replicate + (scale == 1.0))
            p0 = torch.randn(n, device='cuda', generator=gen) * 0.05
            ranks = Ranks(G, n, p0, replicate)
            rev = Ranks(G, n, p0, replicate)
            p_ref, m_ref, v_ref = p0.clone(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
            for step in STEPS:
                what = f'{tag} step {step}'
                grads = rank_grads(G, n, gen)
                pre = ranks.buf['param'][0][:n].clone(), ranks.moments('m'), ranks.moments('v')
                ranks.step(grads, step, scale, range(G))
                rev.step(grads, step, scale, range(G - 1, -1, -1))
                gsum = grads[0].clone()
                for g in grads[1:]:
                    gsum = gsum + g                                     # ((g0 + g1) + g2) + ... in float32
                _lib.check(lib.rlca_adam_step(C.c_void_p(p_ref.data_ptr()), C.c_void_p(gsum.data_ptr()),
                                              C.c_void_p(m_ref.data_ptr()), C.c_void_p(v_ref.data_ptr()), n, LR, BETA1,
                                              BETA2, EPS, step, scale, st))
                torch.cuda.synchronize()
                # 1. bit for bit against the single-GPU kernel
                for q in range(G):
                    if not same_bits(ranks.buf['param'][q][:n], p_ref):
                        check.failed.append(f'{what}: rank {q} parameters differ from rlca_adam_step on the summed '
                                            f'gradient ({first_diff(ranks.buf["param"][q][:n], p_ref)})')
                for k, ref in (('m', m_ref), ('v', v_ref)):
                    got = ranks.moments(k)
                    if not same_bits(got, ref):
                        check.failed.append(f'{what}: {k} differs from rlca_adam_step ({first_diff(got, ref)})')
                    if replicate:
                        for q in range(1, G):
                            if not same_bits(ranks.buf[k][q][:n], ranks.buf[k][0][:n]):
                                check.failed.append(f'{what}: replicated {k} of rank {q} differs from rank 0')
                # 2. float64 Adam within the derived bound
                (p64, m64, v64), (bp, bm, bv) = adam64_with_bound(grads, scale, *pre, step)
                for name, got, ref, b in (('param', ranks.buf['param'][0][:n], p64, bp),
                                          ('m', ranks.moments('m'), m64, bm), ('v', ranks.moments('v'), v64, bv)):
                    r = ratio(got, ref, b)
                    if r > worst.get(name, (-1.0, ''))[0]:
                        worst[name] = (r, what)
                # 3. shards, tails, untouched gradients and launch order
                for q in range(G):
                    for k in Ranks.KINDS:
                        if not same_bits(ranks.buf[k][q][n:], sentinel(TAIL)):
                            check.failed.append(f'{what}: the tail of rank {q} {k} was written')
                        if not same_bits(ranks.buf[k][q], rev.buf[k][q]):
                            check.failed.append(f'{what}: rank {q} {k} differs when the ranks launch in reverse order '
                                                f'({first_diff(ranks.buf[k][q], rev.buf[k][q])})')
                    if not same_bits(ranks.buf['grad'][q][:n], grads[q]):
                        check.failed.append(f'{what}: the gradient of rank {q} was written')
                    if not replicate:
                        lo, hi = kernel_shard(n, G, q)
                        if (lo, hi) != peer_shard(n, G, q):
                            check.failed.append(f'{what}: PeerAdam.shard({q}) = {peer_shard(n, G, q)}, kernel ({lo}, {hi})')
                        for k in ('m', 'v'):
                            written = (bits(ranks.buf[k][q][:n]) != SENTINEL).nonzero().flatten()
                            expect = torch.arange(lo, hi, device='cuda')
                            if not torch.equal(written, expect):
                                span = (int(written[0]), int(written[-1]) + 1) if written.numel() else None
                                check.failed.append(f'{what}: rank {q} wrote {k} at {written.numel()} elements, span '
                                                    f'{span}, not its shard [{lo}, {hi})')
            del ranks, rev
    for name in ('param', 'm', 'v'):
        r, where = worst[name]
        check(f'G={G} n={n} {name} vs float64 Adam (worst: {where})', r, 1.0)
    check.done()


class OneRankPeer:
    """A one-GPU stand-in for parallel.PeerAdam: the fused kernel with G = 1 on the policy's and optimizer's own
    buffers, no multicast, no barriers"""

    def __init__(self, policy):
        self.policy = policy

    def step(self, opt, grad_scale):
        _lib, _, _ = lib_and_stream()
        p = self.policy
        one = lambda t: (C.c_uint64 * 1)(t.data_ptr())
        _lib.check(p.lib.rlca_adam_step_allreduce(one(p.grad), one(p.flat), one(opt.exp_avg), one(opt.exp_avg_sq), 0, 0,
                                                  0, 0, 0, 1, p.flat_size, opt.lr, opt.betas[0], opt.betas[1], opt.eps,
                                                  opt.step_count, grad_scale, 0, p._stream()))


def make_policy(nb, sd):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=nb)
    pol.set_tensor_cores(True)
    pol.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    return pol


def test_adam_peer_branch_refreshes_weight_images(built):
    """Adam.step with `opt.peer` set skips rlca_policy_adam_step, which would have written the tf32 hi / lo split of
    the fc1 weights.  After each such step the tensor-core forward must equal, bit for bit, a fresh policy loaded with
    the new weights (stale fc1 splits or conv images would not), and float64 within the forward bound."""
    from rl_collision_avoidance_b200.model.net import Adam
    _lib, lib, st = lib_and_stream()
    nb = 256
    pool = decisive_pool(nb)
    obs = torch.from_numpy(np.ascontiguousarray(pool['obs'].reshape(nb, 1536))).cuda()
    gs = torch.from_numpy(pool['gs']).cuda()
    pol = make_policy(nb, synthetic_state_dict())
    pol.forward_values(obs, gs)                        # builds the fc1 split and the conv weight image
    opt = Adam(pol.parameters(), lr=1e-3)
    opt.peer = OneRankPeer(pol)
    p_ref, m_ref, v_ref = pol.flat.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone()
    gen = torch.Generator(device='cuda').manual_seed(11)
    check = Checks()
    for step in (1, 2):
        pol.grad.copy_(torch.randn(pol.flat_size, device='cuda', generator=gen) * 0.1)
        _lib.check(lib.rlca_adam_step(C.c_void_p(p_ref.data_ptr()), C.c_void_p(pol.grad.data_ptr()),
                                      C.c_void_p(m_ref.data_ptr()), C.c_void_p(v_ref.data_ptr()), pol.flat_size, opt.lr,
                                      opt.betas[0], opt.betas[1], opt.eps, step, 0.5, st))
        opt.step(grad_scale=0.5)
        v, mean = pol.forward_values(obs, gs)
        torch.cuda.synchronize()
        assert opt.step_count == step
        assert same_bits(pol.flat, p_ref) and same_bits(opt.exp_avg, m_ref) and same_bits(opt.exp_avg_sq, v_ref), \
            f'step {step}: the peer branch differs from rlca_adam_step'
        sd_new = {k: t.cpu().numpy() for k, t in pol.state_dict().items()}
        fresh = make_policy(nb, sd_new)
        v_f, mean_f = fresh.forward_values(obs, gs)
        torch.cuda.synchronize()
        del fresh
        if not (same_bits(v, v_f) and same_bits(mean, mean_f)):
            check.failed.append(f'step {step}: the forward after a peer-branch Adam step differs from a fresh policy '
                                f'with the new weights (max |dv| {float((v - v_f).abs().max()):.3e}, max |dmean| '
                                f'{float((mean - mean_f).abs().max()):.3e}): stale fc1 split or conv image')
        with torch.no_grad():
            v64, mean64, _ = ref_forward(params64(sd_new), obs.double().view(nb, 3, 512), gs.double())
        check_forward(check, f'peer-branch step {step} forward', v, mean, v64, mean64)
    check.done()
