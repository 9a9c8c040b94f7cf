"""The action sampler rlca_policy_sample (sample_kernel, csrc/rlca_policy.cu) against the float64 reference of
tests/sample_ref.py: exact draws at every launch shape, seed and counter word, the log-probability far into the tails,
the distribution and independence of the draws, modes 1 and 2, the scaled clip, CNNPolicy's counter bookkeeping and
the arguments the entry rejects.

Error bounds, with u = 2^-24 the float32 unit roundoff and the maximum errors the CUDA C Programming Guide documents
for the single-precision functions (logf 1 ulp, sincosf 2 ulp, expf 2 ulp; sqrtf and division correctly rounded);
an ulp of x is at most 2u |x|:

* Action, mode 0.  The uniforms and the angle t are exact in both (the reference rounds float32(2 pi) * u2 once, as the
  kernel does).  logf adds 2u relative to ln u1, which sqrtf halves and then rounds (2u on r); sincosf 4u; the
  product r cos t one rounding (u); expf(logstd) 4u; the fmaf with the mean half an ulp of the action.  So
  |a - a_ref| <= 11u sigma |z| + ulp(a) / 2, taken as 12u sigma |z| + ulp(a) / 2 to cover the second-order terms,
  plus 2^-52 |a| for the float64 reference.  That is under 2e-6 (|mean| + sigma |z|) (checked too), while a wrong
  counter, key or word changes a draw by O(sigma), some 10^5 times more.  Where sigma |z| is far below an ulp of the
  action (logstd -5) the bound is the fma's own half-ulp rounding, which one rounding can come within a hair of, so the
  worst ratio there is close to 1 by construction.
* Log-probability, at the kernel's own action (mode 0) or at a given one (modes 1 and 2).  The kernel forms
  ((-(d d) / (2 v) - c) - logstd) per dimension and adds the two, with d = a - mean (u), v = expf(2 logstd) (4u) and c
  the float32 rounding of ln(2 pi) / 2.  The quotient q = d^2 / (2 v) is within 8u q; c is off by a fixed
  |c32 - c| = 1.6e-8 in each dimension; each of the five additions rounds by at most u times its result.  The bound
  is the sum of these, first order in u, times 1.001.  It is a few ulps of the largest term: where the sum cancels,
  as for mode 1 at logstd -1.04 (log-probability 0.24), the fixed error of c alone is 2.1 ulps of the result.

Statistical thresholds sit at about 5 sigma of each statistic: a p-value below 2.9e-7 (the one-sided 5 sigma tail of a
normal) fails, and a Pearson correlation of n pairs fails above 5 / sqrt(n).  The seeds are fixed, so the outcome is
deterministic."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy import stats

import sample_ref as ref
from learner_ref import Checks

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C32_ERR = abs(float(np.float32(ref.LOG_SQRT_2PI)) - ref.LOG_SQRT_2PI)
P_MIN = 2.9e-7
RLCA_ERR_INVALID = 1
POISON = 0x7FC0DEAD                             # a quiet NaN with a payload no kernel writes

NBS = (1, 127, 128, 129, 4104, 65544)            # block edges, the 171 x 24 rollout, the raycast-sweep size
SEEDS = (0, 1, 2 ** 32, 2 ** 64 - 1)            # 2^32: only the high key word is set
COUNTERS = (1, 2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1)   # 2^32: the carry into the third counter word
LOGSTDS = (-5.0, -1.85, -1.04, 0.0, 2.0)         # the shipped checkpoints have logstd in [-1.85, -1.04]
LS_PAIRS = tuple((LOGSTDS[k], LOGSTDS[(k + 2) % 5]) for k in range(5))   # every value in both dimensions, never equal


def _lib():
    from rl_collision_avoidance_b200 import _lib as lib
    return lib.load()


def ptr(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def params_with(logstd):
    """a parameter buffer holding only what the sampler reads: logstd at its offset in the flat layout"""
    lib = _lib()
    assert int(lib.rlca_policy_param_size(0)) == 2
    o = int(lib.rlca_policy_param_offset(0))
    p = torch.zeros(int(lib.rlca_policy_param_offset(1)), device='cuda')
    p[o:o + 2] = torch.from_numpy(np.float32(logstd)).cuda()
    return p


def spread_means(n, seed):
    rs = np.random.RandomState(seed)
    return np.stack([rs.uniform(0, 1, n), rs.uniform(-1, 1, n)], 1).astype(np.float32)


def call(params, mean, seed, counter, mode, action, logprob, scaled=None, nb=None):
    return _lib().rlca_policy_sample(ptr(params), ptr(mean), mean.shape[0] if nb is None else nb, seed, counter, mode,
                                     ptr(action), ptr(logprob), ptr(scaled), None)


def draw(params, mean_d, seed, counter, mode=0, action=None):
    """(action, logprob, scaled) of one call as numpy; mode 2 evaluates `action` (numpy)"""
    nb = mean_d.shape[0]
    act = torch.empty(nb, 2, device='cuda') if action is None else torch.from_numpy(np.ascontiguousarray(action)).cuda()
    lp = torch.empty(nb, device='cuda')
    sc = torch.empty(nb, 2, device='cuda')
    assert call(params, mean_d, seed, counter, mode, act, lp, sc) == 0
    return act.cpu().numpy(), lp.cpu().numpy(), sc.cpu().numpy()


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def action_bound(a, sz):
    """12u sigma |z| + half an ulp of the float32 action (module docstring), + 2^-52 |a| for the float64 reference"""
    a = np.abs(np.float32(a))
    return 12 * U * sz + np.spacing(a).astype(np.float64) / 2 + 2.0 ** -52 * a


def lp_bound(a, mean, logstd):
    """the log-probability bound of the module docstring at the float32 action a"""
    d = np.float64(a) - np.float64(mean)
    ls = np.float64(np.float32(logstd))
    q = d * d / (2 * np.exp(2 * ls))
    p1 = -q - ref.LOG_SQRT_2PI
    p2 = p1 - ls
    s = p2.sum(-1)
    return 1.001 * (8 * U * q.sum(-1) + 2 * C32_ERR + U * (np.abs(p1).sum(-1) + np.abs(p2).sum(-1) + np.abs(s)))


class Worst:
    """the largest error / bound ratio over many rows, and where it was"""

    def __init__(self):
        self.ratio, self.err, self.bound, self.where = -1.0, 0.0, 1.0, ''

    def add(self, err, bound, where):
        assert np.isfinite(err).all(), where
        r = err / bound
        i = int(np.argmax(r))
        if r.flat[i] > self.ratio:
            self.ratio, self.err, self.bound = float(r.flat[i]), float(err.flat[i]), float(bound.flat[i])
            self.where = f'{where}, row {i}'

    def report(self, check, what):
        check(f'{what} (worst: {self.where})', self.err, self.bound)


def corr_check(check, what, x, y):
    x, y = np.ravel(x), np.ravel(y)
    check(f'correlation {what}', abs(float(np.corrcoef(x, y)[0, 1])), 5 / math.sqrt(len(x)))


def p_check(check, what, p):
    """fails below P_MIN; prints P_MIN / p"""
    check(f'{what} p-value {p:.3g}', P_MIN, p)


# ------------------------------------------------------------------------------------------------ mode 0
def test_exact_draws_at_every_shape_seed_and_counter(built):
    """Mode 0 against the reference at every nb, seed, counter and logstd pair: the action to the bound of the module
    docstring (which itself stays under 2e-6 (|mean| + sigma |z|)), the log-probability at the kernel's own action to
    its bound, and the scaled action is the float32 clip of the action bit for bit."""
    check = Checks()
    means = spread_means(max(NBS), 1)
    mean_d = torch.from_numpy(means).cuda()
    params = {ls: params_with(ls) for ls in LS_PAIRS}
    for seed in SEEDS:
        for counter in COUNTERS:
            z = ref.normals(seed, counter, max(NBS))
            wa, wl, wc = Worst(), Worst(), Worst()
            for ls in LS_PAIRS:
                sig = ref.sigma(ls)
                for nb in NBS:
                    act, lp, sc = draw(params[ls], mean_d[:nb], seed, counter)
                    where = f'logstd {ls}, nb {nb}'
                    m64, sz = np.float64(means[:nb]), sig * np.abs(z[:nb])
                    bound = action_bound(act, sz)
                    wa.add(np.abs(act - (m64 + sig * z[:nb])), bound, where)
                    wc.add(bound, 2e-6 * (np.abs(m64) + sz), where)
                    wl.add(np.abs(lp - ref.log_prob(act, means[:nb], ls)), lp_bound(act, means[:nb], ls), where)
                    assert np.array_equal(bits(sc), bits(ref.scaled(act))), (seed, counter, where)
            what = f'seed {seed:#x} counter {counter:#x}'
            wa.report(check, f'{what} action')
            wc.report(check, f'{what} action bound / 2e-6 (|mean| + sigma |z|)')
            wl.report(check, f'{what} logprob')
    check.done()


def test_draw_depends_only_on_seed_counter_and_row(built):
    """row i of an nb = 65544 call is bit-identical to row i of calls with nb = 1, 129 and 4104: no draw depends on
    the grid, the block or the batch size"""
    means = spread_means(max(NBS), 2)
    mean_d = torch.from_numpy(means).cuda()
    params = params_with((-1.85, -1.04))
    for seed, counter in ((0, 1), (2 ** 32, 2 ** 32 - 1), (2 ** 64 - 1, 2 ** 32), (12345, 2 ** 64 - 1)):
        big = draw(params, mean_d, seed, counter)
        for nb in (1, 129, 4104):
            small = draw(params, mean_d[:nb], seed, counter)
            for b, s in zip(big, small):
                assert np.array_equal(bits(b[:nb]), bits(s)), (seed, counter, nb)


def _z_block(params, mean_d, means, sig, seed, counters):
    """(len(counters), nb, 2) float64 normals recovered from the kernel's actions, z = (a - mean) / sigma"""
    nb = mean_d.shape[0]
    act = torch.empty(len(counters), nb, 2, device='cuda')
    lp = torch.empty(len(counters), nb, device='cuda')
    for k, c in enumerate(counters):
        assert call(params, mean_d, seed, c, 0, act[k], lp[k]) == 0
    return (act.cpu().numpy().astype(np.float64) - np.float64(means)) / sig


def test_distribution_and_independence(built):
    """About 10^6 pairs (4104 rows x 256 counters) at fixed seeds, z = (a - mean) / sigma: Kolmogorov-Smirnov of each
    dimension against N(0, 1), of r^2 against chi^2 with 2 degrees of freedom and of the angle against uniform; a
    16 x 16 equal-probability binned chi^2 of (z0, z1); and no Pearson correlation between the two dimensions of a
    row, adjacent rows, counters k and k + 1, counters k and k + 2^32, seeds s and s + 1 (two ranks) or seeds s and
    s + 2^32."""
    check = Checks()
    nb, seed, ls = 4104, 0x5EED_2024, (-1.04, -1.85)
    counters = np.arange(1, 257, dtype=np.uint64)
    means = spread_means(nb, 3)
    mean_d = torch.from_numpy(means).cuda()
    params, sig = params_with(ls), ref.sigma(ls)
    A = _z_block(params, mean_d, means, sig, seed, [int(c) for c in counters])
    z0, z1 = A[..., 0].ravel(), A[..., 1].ravel()
    p_check(check, 'KS z0 ~ N(0, 1)', stats.kstest(z0, 'norm').pvalue)
    p_check(check, 'KS z1 ~ N(0, 1)', stats.kstest(z1, 'norm').pvalue)
    p_check(check, 'KS r^2 ~ chi2(2)', stats.kstest(z0 * z0 + z1 * z1, 'chi2', args=(2,)).pvalue)
    p_check(check, 'KS angle ~ U(0, 2 pi)', stats.kstest(np.arctan2(z1, z0) % (2 * np.pi) / (2 * np.pi), 'uniform').pvalue)
    cell = np.minimum((stats.norm.cdf(A) * 16).astype(np.int64), 15)
    counts = np.bincount((cell[..., 0] * 16 + cell[..., 1]).ravel(), minlength=256)
    expect = z0.size / 256
    p_check(check, 'binned chi^2 of (z0, z1)', stats.chi2.sf(((counts - expect) ** 2 / expect).sum(), 255))

    corr_check(check, 'z0, z1 of a row', z0, z1)
    for d in (0, 1):
        corr_check(check, f'adjacent rows, dim {d}', A[:, :-1, d], A[:, 1:, d])
        corr_check(check, f'counter k, k + 1, dim {d}', A[:-1, :, d], A[1:, :, d])
    others = {'counter k, k + 2^32': (seed, counters + np.uint64(2 ** 32)),
              'seed s, s + 1': (seed + 1, counters), 'seed s, s + 2^32': (seed + 2 ** 32, counters)}
    for what, (s, cs) in others.items():
        B = _z_block(params, mean_d, means, sig, s, [int(c) for c in cs])
        for d in (0, 1):
            corr_check(check, f'{what}, dim {d}', A[..., d], B[..., d])
        corr_check(check, f'{what}, dim 0 against dim 1', A[..., 0], B[..., 1])
    check.done()


# ------------------------------------------------------------------------------------------------ modes 1 and 2, clip
def _edge_actions():
    """actions on the bound [[0, -1], [1, 1]], one float32 step inside and outside it, and beyond it"""
    nx = lambda x, to: np.nextafter(np.float32(x), np.float32(to))
    e0 = [0.0, 1.0, nx(0, -1), nx(0, 1), nx(1, 0), nx(1, 2), -3.5, 0.5, 7.25]
    e1 = [-1.0, 1.0, nx(-1, -2), nx(-1, 0), nx(1, 0), nx(1, 2), -9.0, 0.0, 3.0]
    return np.array([(a, b) for a in e0 for b in e1], np.float32)


def test_mode1_returns_the_mean(built):
    """Mode 1: the action is the mean bit for bit, whatever the seed and counter, the log-probability is
    -sum(ln(2 pi) / 2 + logstd) within the bound of the module docstring at d = 0, and scaled is the clip of the mean
    bit for bit, the bound's edges included."""
    check = Checks()
    means = np.concatenate([_edge_actions(), spread_means(4104 - 81, 4)])
    mean_d = torch.from_numpy(means).cuda()
    for ls in LS_PAIRS + tuple((v, v) for v in LOGSTDS):
        params = params_with(ls)
        first = None
        for seed, counter in ((0, 1), (2 ** 64 - 1, 2 ** 32)):
            act, lp, sc = draw(params, mean_d, seed, counter, 1)
            assert np.array_equal(bits(act), bits(means)), ls
            assert np.array_equal(bits(sc), bits(ref.scaled(means))), ls
            if first is None:
                first = lp
            assert np.array_equal(bits(lp), bits(first)), ls
        want = -2 * ref.LOG_SQRT_2PI - float(np.float64(np.float32(ls)).sum())
        err = np.abs(np.float64(lp) - want)
        check(f'mode 1 logprob, logstd {ls} ({err.max() / np.spacing(np.float32(abs(want))):.2f} ulp)', err.max(),
              float(lp_bound(means[:1] * 0, means[:1] * 0, ls)[0]))
    check.done()


def test_mode2_evaluates_given_actions_into_the_tails(built):
    """Mode 2 at actions |a - mean| / sigma from 0 to 40 and on the clip's edges: the log-probability within its bound
    of float64, the action buffer unchanged bit for bit, scaled the clip of the given action bit for bit; an infinite
    action gives -inf and clips to the bound."""
    check = Checks()
    n = 4096
    rs = np.random.RandomState(5)
    means = spread_means(n, 6)
    k = np.linspace(0, 40, n)[:, None] * rs.choice([-1.0, 1.0], (n, 2))
    rs.shuffle(k)
    edges = _edge_actions()
    inf = np.array([[np.inf, 0.5], [-np.inf, 0.5], [0.5, np.inf], [0.5, -np.inf], [np.inf, -np.inf]], np.float32)
    for ls in LS_PAIRS:
        a = np.concatenate([np.float32(means + ref.sigma(ls) * k), edges, inf])
        m = np.concatenate([means, spread_means(len(edges) + len(inf), 7)])
        act, lp, sc = draw(params_with(ls), torch.from_numpy(m).cuda(), 3, 4, 2, action=a)
        assert np.array_equal(bits(act), bits(a)), ls
        assert np.array_equal(bits(sc), bits(ref.scaled(a))), ls
        fin = slice(0, n + len(edges))
        w = Worst()
        w.add(np.abs(np.float64(lp[fin]) - ref.log_prob(a[fin], m[fin], ls)), lp_bound(a[fin], m[fin], ls), 'rows')
        w.report(check, f'mode 2 logprob, logstd {ls}')
        assert (lp[n + len(edges):] == -np.inf).all(), lp[n + len(edges):]
    check.done()


def test_scaled_clip_in_mode0_and_null_scaled(built):
    """Mode 0 at logstd 2 around means on the bound's edges: scaled is the float32 clip of the drawn action bit for bit
    (and the draws do leave the bound on both sides of both dimensions).  In every mode the entry writes exactly its
    nb-row slices of action, logprob and scaled; with scaled NULL a poisoned buffer after logprob stays untouched."""
    edges = _edge_actions()
    means = np.concatenate([edges] * 16)
    act, _, sc = draw(params_with((2.0, 2.0)), torch.from_numpy(means).cuda(), 99, 7)
    assert np.array_equal(bits(sc), bits(ref.scaled(act)))
    for d, (lo, hi) in enumerate(((0.0, 1.0), (-1.0, 1.0))):
        assert (act[:, d] < lo).any() and (act[:, d] > hi).any() and ((act[:, d] > lo) & (act[:, d] < hi)).any()

    nb, g = 129, 64
    means = spread_means(nb, 8)
    mean_d = torch.from_numpy(means).cuda()
    params = params_with((-1.85, -1.04))
    o_act, o_lp = g, g + 2 * nb + g
    o_sc = o_lp + nb + g
    total = o_sc + 2 * nb + g
    given = np.float32(means + 0.25)
    for mode in (0, 1, 2):
        for with_scaled in (False, True):
            arena = torch.full((total,), POISON, dtype=torch.int32, device='cuda').view(torch.float32)
            if mode == 2:
                arena[o_act:o_act + 2 * nb] = torch.from_numpy(given.ravel()).cuda()
            act, lp = arena[o_act:o_act + 2 * nb], arena[o_lp:o_lp + nb]
            sc = arena[o_sc:o_sc + 2 * nb] if with_scaled else None
            assert call(params, mean_d, 1, 1, mode, act, lp, sc) == 0
            out = arena.cpu().numpy()
            written = np.zeros(total, bool)
            written[o_act:o_act + 2 * nb] = written[o_lp:o_lp + nb] = True
            if with_scaled:
                written[o_sc:o_sc + 2 * nb] = True
                assert np.array_equal(bits(out[o_sc:o_sc + 2 * nb]), bits(ref.scaled(out[o_act:o_act + 2 * nb]
                                                                                      .reshape(nb, 2)).ravel()))
            assert (bits(out[~written]) == POISON).all(), (mode, with_scaled)
            assert np.isfinite(out[written]).all(), (mode, with_scaled)


def test_rejected_arguments_leave_outputs_untouched(built):
    """deterministic -1 or 3, nb = 0 and a NULL mean, action or logprob return RLCA_ERR_INVALID and launch nothing:
    the poisoned output buffers keep their bits"""
    nb = 129
    mean_d = torch.from_numpy(spread_means(nb, 9)).cuda()
    params = params_with((0.0, 0.0))
    act, lp, sc = (torch.full((m,), POISON, dtype=torch.int32, device='cuda').view(torch.float32)
                   for m in (2 * nb, nb, 2 * nb))
    bad = [dict(mode=-1), dict(mode=3), dict(nb=0), dict(mean=None), dict(action=None), dict(logprob=None)]
    for kw in bad:
        for mode in ((kw['mode'],) if 'mode' in kw else (0, 1, 2)):
            args = dict(params=params, mean=mean_d, action=act, logprob=lp)
            args.update({k: v for k, v in kw.items() if k in args})
            rc = _lib().rlca_policy_sample(ptr(args['params']), ptr(args['mean']), kw.get('nb', nb), 1, 1, mode,
                                           ptr(args['action']), ptr(args['logprob']), ptr(sc), None)
            assert rc == RLCA_ERR_INVALID, (kw, mode)
    torch.cuda.synchronize()
    for t in (act, lp, sc):
        assert (bits(t.cpu().numpy()) == POISON).all()


# ------------------------------------------------------------------------------------------------ CNNPolicy
def _policy(nb, logstd, seed):
    from golden_inputs import synthetic_state_dict
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=nb)
    sd = synthetic_state_dict()
    sd['logstd'] = np.float32(logstd)
    pol.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    pol.sample_seed = seed
    return pol


def _inputs(nb):
    from golden_inputs import synthetic_batch
    obs, goal, speed, action = synthetic_batch(64, seed=13)
    rep = lambda x: torch.from_numpy(np.ascontiguousarray(np.resize(x, (nb,) + x.shape[1:]))).cuda()
    return rep(obs), rep(goal), rep(speed), rep(action)


def test_policy_counter_and_resume(built):
    """forward advances sample_counter by exactly one and draws at the advanced value (equal to the reference within
    the action bound); evaluate_actions leaves it alone.  A fresh policy with the same weights, seed and counter draws
    the same bits: what --resume relies on through the sample_counter saved in .trainer."""
    check = Checks()
    nb, ls, seed = 1000, (-1.85, -1.04), 2 ** 40 + 3
    x, goal, speed, given = _inputs(nb)
    pol = _policy(nb, ls, seed)
    assert pol.sample_counter == 0
    w = Worst()
    for step in range(1, 4):
        _, a, lp, mean = pol(x, goal, speed)
        assert pol.sample_counter == step
        a, mean = a.cpu().numpy(), mean.cpu().numpy()
        z = ref.normals(seed, step, nb)
        sig = ref.sigma(ls)
        w.add(np.abs(a - (np.float64(mean) + sig * z)), action_bound(a, sig * np.abs(z)), f'call {step}')
        pol.evaluate_actions(x, goal, speed, given)
        assert pol.sample_counter == step
    w.report(check, 'CNNPolicy.forward action')

    twin = _policy(nb, ls, seed)
    twin.sample_counter = pol.sample_counter
    for _ in range(2):
        got = [t.cpu().numpy() for t in pol(x, goal, speed)]
        want = [t.cpu().numpy() for t in twin(x, goal, speed)]
        for g, t in zip(got, want):
            assert np.array_equal(bits(g), bits(t))
    assert twin.sample_counter == pol.sample_counter == 5
    check.done()


def test_ranks_draw_uncorrelated_noise(built):
    """ranks 0 and 1 of a data-parallel run (sample_seed = seed * 1000003 + rank, ppo_stage1.py) draw uncorrelated
    noise on the same inputs, call after call"""
    check = Checks()
    nb, calls, ls = 4104, 64, (-1.04, -1.85)
    x, goal, speed, _ = _inputs(nb)
    sig = ref.sigma(ls)
    z = []
    for rank in (0, 1):
        pol = _policy(nb, ls, 7 * 1000003 + rank)
        zs = []
        for _ in range(calls):
            _, a, _, mean = pol(x, goal, speed)
            zs.append((a.cpu().numpy().astype(np.float64) - mean.cpu().numpy()) / sig)
        z.append(np.stack(zs))
    for d in (0, 1):
        corr_check(check, f'rank 0, rank 1, dim {d}', z[0][..., d], z[1][..., d])
    corr_check(check, 'rank 0 dim 0, rank 1 dim 1', z[0][..., 0], z[1][..., 1])
    check.done()
