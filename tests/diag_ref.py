"""Float64 numpy reference of the PPO update diagnostics (DESIGN.md §9n): every accumulator column of
rlca_ppo_diag_accumulate and rlca_grad_sumsq, the metrics computed from them, and the decisive batches the tests use.

Decisive batches: every PPO ratio is at least MARGIN away from 1 +- clip and every policy mean and sampled action at
least MARGIN away from the action bound, so fp32 rounding cannot move a row across a threshold and the counts of the
kernel and of the float64 reference must be equal."""
import math

import numpy as np

MARGIN = 1e-5
CLIP = 0.1
BOUND = ((0.0, -1.0), (1.0, 1.0))
LOGSTD = (-0.3, 0.2)
LOG_2PI_HALF = 0.5 * math.log(2 * math.pi)

SUM_COLUMNS = ('n', 'sum_kl', 'sum_kl_k3', 'clipped', 'cut', 'sum_ratio', 'sum_err', 'sum_err_sq', 'sum_target',
               'sum_target_sq', 'sum_value', 'sum_adv', 'sum_adv_sq', 'mean_out_0', 'mean_out_1', 'action_out_0',
               'action_out_1')
COUNT_COLUMNS = ('n', 'clipped', 'cut', 'mean_out_0', 'mean_out_1', 'action_out_0', 'action_out_1')


def logprob64(logstd, mean, action):
    ls = np.asarray(logstd, dtype=np.float64)
    d = action.astype(np.float64) - mean.astype(np.float64)
    return (-(d * d) / (2 * np.exp(2 * ls)) - LOG_2PI_HALF - ls).sum(1)


def ratio32(logstd, mean, action, old_lp):
    """The ratio in the kernel's fp32 arithmetic, operation by operation.  Only the two exp calls (of 2 logstd and of
    the log-ratio) are not bit-defined: the device's expf is within 2 ulp of the rounded exact value, which moves the
    ratio by a few ulp."""
    f = np.float32
    ls = np.asarray(logstd, dtype=f)
    var = np.exp((f(2.0) * ls).astype(np.float64)).astype(f)
    d = action.astype(f) - mean.astype(f)
    terms = -(d * d) / (f(2.0) * var) - f(LOG_2PI_HALF) - ls
    logr = (terms[:, 0] + terms[:, 1]) - old_lp.astype(f)
    return np.exp(logr.astype(np.float64)).astype(f)


def decisive_batch(rs, n, clip=CLIP, bound=BOUND, logstd=LOGSTD, spread=0.25):
    """n decisive rows: value, mean (n, 2), action (n, 2), old_lp, adv, target as float32.  Means and actions reach
    beyond the bound, and exp(+-spread) beyond 1 +- clip, so every count is exercised."""
    (lo0, lo1), (hi0, hi1) = bound
    out = {k: [] for k in ('value', 'mean', 'action', 'old_lp', 'adv', 'target')}
    have = 0
    while have < n:
        m = 2 * n + 16
        mean = np.stack([rs.uniform(lo0 - 0.1, hi0 + 0.1, m), rs.uniform(lo1 - 0.1, hi1 + 0.1, m)], 1).astype(np.float32)
        action = np.stack([rs.uniform(lo0 - 0.2, hi0 + 0.2, m), rs.uniform(lo1 - 0.2, hi1 + 0.2, m)], 1).astype(np.float32)
        old_lp = (logprob64(logstd, mean, action) - rs.uniform(-spread, spread, m)).astype(np.float32)
        ratio = np.exp(logprob64(logstd, mean, action) - old_lp.astype(np.float64))
        ok = (np.abs(ratio - (1 - clip)) >= MARGIN) & (np.abs(ratio - (1 + clip)) >= MARGIN)
        for x in (mean, action):
            for k, (lo, hi) in enumerate(((lo0, hi0), (lo1, hi1))):
                ok &= (np.abs(x[:, k].astype(np.float64) - lo) >= MARGIN) & (np.abs(x[:, k].astype(np.float64) - hi) >= MARGIN)
        d = dict(value=rs.uniform(-3, 3, m), mean=mean, action=action, old_lp=old_lp, adv=rs.standard_normal(m),
                 target=rs.uniform(-3, 3, m))
        for k in out:
            out[k].append(np.asarray(d[k], dtype=np.float32)[ok])
        have += int(ok.sum())
    return {k: np.concatenate(v)[:n] for k, v in out.items()}


def ref_row(b, clip=CLIP, bound=BOUND, logstd=LOGSTD):
    """(columns, scales) of the minibatch b: every column of rlca_ppo_diag_accumulate in float64 from the fp32 inputs,
    and for every sum column the sum of the magnitudes of its terms plus the row count - the scale its error is held
    against."""
    (lo0, lo1), (hi0, hi1) = bound
    v, t, A = (b[k].astype(np.float64) for k in ('value', 'target', 'adv'))
    logr = logprob64(logstd, b['mean'], b['action']) - b['old_lp'].astype(np.float64)
    r = np.exp(logr)
    m, a = b['mean'].astype(np.float64), b['action'].astype(np.float64)
    outside = lambda x, lo, hi: (~((x > lo) & (x < hi))).astype(np.float64)
    terms = {
        'n': np.ones_like(r), 'sum_kl': -logr, 'sum_kl_k3': (r - 1) - logr,
        'clipped': (np.abs(r - 1) > clip).astype(np.float64),
        'cut': (((r > 1 + clip) & (A > 0)) | ((r < 1 - clip) & (A < 0))).astype(np.float64),
        'sum_ratio': r, 'sum_err': t - v, 'sum_err_sq': (t - v) ** 2, 'sum_target': t, 'sum_target_sq': t * t,
        'sum_value': v, 'sum_adv': A, 'sum_adv_sq': A * A,
        'mean_out_0': outside(m[:, 0], lo0, hi0), 'mean_out_1': outside(m[:, 1], lo1, hi1),
        'action_out_0': outside(a[:, 0], lo0, hi0), 'action_out_1': outside(a[:, 1], lo1, hi1),
    }
    cols = {k: float(x.sum()) for k, x in terms.items()}
    cols['max_ratio'], cols['min_ratio'] = float(r.max()), float(r.min())
    scales = {k: float(np.abs(x).sum()) + len(r) for k, x in terms.items()}
    return cols, scales


def union(batches):
    return {k: np.concatenate([b[k] for b in batches]) for k in batches[0]}


def ref_grad_sumsq(grad, offsets, sizes):
    """Sum of g^2 of every tensor of a flat gradient buffer, padding excluded, in float64."""
    g = np.asarray(grad, dtype=np.float64)
    return np.array([float((g[o:o + n] ** 2).sum()) for o, n in zip(offsets, sizes)])


def ref_metrics(c):
    """The metrics of DESIGN.md §9n from a dict of merged minibatch columns, written out independently of the product."""
    n = c['n']
    var = lambda s, ss: max(ss / n - (s / n) ** 2, 0.0)
    var_t = var(c['sum_target'], c['sum_target_sq'])
    return {
        'approx_kl': c['sum_kl'] / n, 'approx_kl_k3': c['sum_kl_k3'] / n,
        'clip_fraction': c['clipped'] / n, 'cut_fraction': c['cut'] / n,
        'ratio_mean': c['sum_ratio'] / n, 'ratio_max': c['max_ratio'], 'ratio_min': c['min_ratio'],
        'explained_variance': 1 - var(c['sum_err'], c['sum_err_sq']) / var_t if var_t > 0 else float('nan'),
        'value_rmse': math.sqrt(c['sum_err_sq'] / n), 'value_bias': (c['sum_value'] - c['sum_target']) / n,
        'adv_mean': c['sum_adv'] / n, 'adv_std': math.sqrt(var(c['sum_adv'], c['sum_adv_sq'])),
        'mean_saturation': [c['mean_out_0'] / n, c['mean_out_1'] / n],
        'action_saturation': [c['action_out_0'] / n, c['action_out_1'] / n],
    }
