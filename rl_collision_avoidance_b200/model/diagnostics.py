"""How healthy a PPO update is (DESIGN.md §9n): approximate KL, clip fraction, explained variance, ratio extremes,
action saturation and gradient norms.

The per-minibatch tensors live on the device and are overwritten every minibatch, so two librlca.so kernels accumulate
what the metrics need into one float64 row per epoch (rlca_ppo_diag_accumulate, rlca_grad_sumsq); the rows come back in
one D2H per update and `metrics` turns them into numbers on the host.  Every column has one merge rule - sum, max or
min - so minibatches, epochs and data-parallel ranks combine by that rule (`merge_rows`, parallel.allreduce_diagnostics).
"""
from __future__ import annotations

import ctypes as C
import logging
import math
import os
import socket

import numpy as np
import torch

from .. import _lib
from .net import TENSORS, _ptr

logger_diag = logging.getLogger('loggerdiag')

# the RLCA_PPO_DIAG_* columns of include/rlca.h: (name, merge rule)
COLUMNS = ([('n', 'sum'), ('sum_kl', 'sum'), ('sum_kl_k3', 'sum'), ('clipped', 'sum'), ('cut', 'sum'),
            ('sum_ratio', 'sum'), ('sum_err', 'sum'), ('sum_err_sq', 'sum'), ('sum_target', 'sum'),
            ('sum_target_sq', 'sum'), ('sum_value', 'sum'), ('sum_adv', 'sum'), ('sum_adv_sq', 'sum'),
            ('mean_out_0', 'sum'), ('mean_out_1', 'sum'), ('action_out_0', 'sum'), ('action_out_1', 'sum'),
            ('max_ratio', 'max'), ('min_ratio', 'min'), ('grad_steps', 'sum')]
           + [('grad_sumsq.' + name, 'sum') for name, _ in TENSORS] + [('max_grad_sumsq', 'max')])
NAMES = [name for name, _ in COLUMNS]
RULES = [rule for _, rule in COLUMNS]
COL = {name: i for i, name in enumerate(NAMES)}
EMPTY_ROW = np.array([{'sum': 0.0, 'max': -math.inf, 'min': math.inf}[r] for r in RULES])

GROUPS = ('actor_conv', 'critic_conv', 'actor_fc', 'critic_fc', 'heads', 'logstd')


def tensor_group(name):
    """The gradient-norm group of a state_dict tensor."""
    if name == 'logstd':
        return 'logstd'
    layer = name.rsplit('.', 1)[0]
    if layer in ('actor1', 'actor2', 'critic'):
        return 'heads'
    tower = {'act': 'actor', 'crt': 'critic'}[layer[:3]]
    return tower + ('_conv' if '_fea_cv' in layer else '_fc')


def setup_diag_log(root='./log'):
    """./log/<hostname>/diag.log beside ppo.log: one line per update."""
    d = os.path.join(root, socket.gethostname())
    os.makedirs(d, exist_ok=True)
    logger_diag.setLevel(logging.INFO)
    if not logger_diag.handlers:
        h = logging.FileHandler(os.path.join(d, 'diag.log'), mode='a')
        h.setLevel(logging.INFO)
        logger_diag.addHandler(h)
    return logger_diag


def check_target_kl(x):
    """The KL threshold of the stop rule as a float; ValueError unless it is finite and > 0."""
    x = float(x)
    if not (math.isfinite(x) and x > 0):
        raise ValueError('the target KL must be finite and > 0, got %r' % x)
    return x


def merge_rows(rows):
    """Rows (k, COLUMNS) of minibatches, epochs or ranks merged into one, each column by its rule."""
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, len(COLUMNS))
    if not len(rows):
        return EMPTY_ROW.copy()
    op = {'sum': np.sum, 'max': np.max, 'min': np.min}
    return np.array([op[rule](rows[:, c]) for c, rule in enumerate(RULES)])


def _row_metrics(row):
    nan = float('nan')
    g = lambda name: float(row[COL[name]])
    n, steps = g('n'), g('grad_steps')
    m = {'rows': int(n)}
    per_row = lambda name: g(name) / n if n else nan
    m['approx_kl'] = per_row('sum_kl')
    m['approx_kl_k3'] = per_row('sum_kl_k3')
    m['clip_fraction'] = per_row('clipped')
    m['cut_fraction'] = per_row('cut')
    m['ratio_mean'] = per_row('sum_ratio')
    m['ratio_max'] = g('max_ratio') if n else nan
    m['ratio_min'] = g('min_ratio') if n else nan
    var = lambda s, ss: max(g(ss) / n - (g(s) / n) ** 2, 0.0) if n else nan
    var_err, var_t = var('sum_err', 'sum_err_sq'), var('sum_target', 'sum_target_sq')
    # a constant target leaves rounding noise in the float64 moments, not an exact 0
    flat = not n or var_t <= 1e-12 * g('sum_target_sq') / n
    m['explained_variance'] = nan if flat else 1.0 - var_err / var_t
    m['value_rmse'] = math.sqrt(per_row('sum_err_sq')) if n else nan
    m['value_bias'] = (g('sum_value') - g('sum_target')) / n if n else nan
    m['adv_mean'] = per_row('sum_adv')
    m['adv_std'] = math.sqrt(var('sum_adv', 'sum_adv_sq')) if n else nan
    m['mean_saturation'] = [per_row('mean_out_0'), per_row('mean_out_1')]
    m['action_saturation'] = [per_row('action_out_0'), per_row('action_out_1')]
    by_group = dict.fromkeys(GROUPS, 0.0)
    for name, _ in TENSORS:
        by_group[tensor_group(name)] += g('grad_sumsq.' + name)
    m['grad_norm'] = math.sqrt(sum(by_group.values()) / steps) if steps else nan
    m['grad_norm_max'] = math.sqrt(g('max_grad_sumsq')) if steps else nan
    m['grad_norm_by_group'] = {k: math.sqrt(v / steps) if steps else nan for k, v in by_group.items()}
    return m


def metrics(acc):
    """The metrics of merged accumulator rows (epochs, COLUMNS): those of the whole update, and under 'per_epoch' the
    same of every epoch.  A row without minibatches gives NaN.
      approx_kl, approx_kl_k3        mean of old_lp - new_lp, and of (r - 1) - log r, whose terms are not negative
      clip_fraction, cut_fraction    rows with |r - 1| > clip; rows whose surrogate gradient the clip zeroes
      ratio_mean, ratio_max, ratio_min
      explained_variance             1 - Var(t - V) / Var(t), NaN when the targets do not vary
      value_rmse, value_bias         root mean square of t - V; mean of V - t
      adv_mean, adv_std              of the normalised advantages the minibatches saw
      mean_saturation, action_saturation     per action dimension, rows whose policy mean / sampled action is not
                                     strictly inside the action bound
      grad_norm, grad_norm_max       root of the mean, and of the largest, minibatch sum of g^2 over the whole buffer
      grad_norm_by_group             the same root mean per group of tensors (GROUPS)
    The gradient is the one the backward wrote on this rank (rlca_grad_sumsq), before any exchange."""
    acc = np.asarray(acc, dtype=np.float64).reshape(-1, len(COLUMNS))
    out = _row_metrics(merge_rows(acc))
    out['per_epoch'] = [_row_metrics(r) for r in acc]
    return out


def over_target_kl(row, target_kl):
    """The stop rule: True when the epoch whose merged row this is moved the policy by more than target_kl
    (approx_kl_k3), or by a KL that is not a number.  An epoch without rows never stops the update."""
    m = _row_metrics(row)
    return m['rows'] > 0 and not m['approx_kl_k3'] <= target_kl


def format_line(update, m):
    """The diag.log line of an update."""
    pair = lambda v: '(%.4f, %.4f)' % tuple(v)
    groups = ', '.join('%s %.4g' % (k, v) for k, v in m['grad_norm_by_group'].items())
    return ('update %d, epochs %d, rows %d, kl %.6f, kl_k3 %.6f, clip %.4f, cut %.4f, ratio %.4f [%.4f, %.4f], '
            'ev %.4f, value rmse %.4f bias %.4f, adv %.4f +- %.4f, saturation mean %s action %s, logstd %s, '
            'grad norm %.4g max %.4g, %s' %
            (update, m['epochs_run'], m['rows'], m['approx_kl'], m['approx_kl_k3'], m['clip_fraction'],
             m['cut_fraction'], m['ratio_mean'], m['ratio_min'], m['ratio_max'], m['explained_variance'],
             m['value_rmse'], m['value_bias'], m['adv_mean'], m['adv_std'], pair(m['mean_saturation']),
             pair(m['action_saturation']), pair(m['logstd']), m['grad_norm'], m['grad_norm_max'], groups))


class PPODiagnostics:
    """The accumulator rows of one policy's updates, one row per epoch, on the policy's device.

        diag = PPODiagnostics(policy, epochs, action_bound)
        ppo_update_stage2(..., diagnostics=diag, target_kl=0.02)      # resets, accumulates, sets diag.epochs_run
        m = diag.metrics()
    """

    def __init__(self, policy, epochs, action_bound):
        if epochs < 1:
            raise ValueError('diagnostics need at least one epoch, got %d' % epochs)
        self.policy, self.epochs = policy, int(epochs)
        lo, hi = action_bound
        self.bound = (C.c_float * 4)(float(lo[0]), float(lo[1]), float(hi[0]), float(hi[1]))
        self._empty = torch.from_numpy(EMPTY_ROW).to(policy.device)
        self.acc = torch.empty(self.epochs, len(COLUMNS), dtype=torch.float64, device=policy.device)
        self.reset()

    def reset(self):
        self.acc.copy_(self._empty.expand_as(self.acc))
        self.epochs_run = 0

    def accumulate(self, epoch, value, mean, action, old_logprob, adv, target, nb, clip_value):
        """One minibatch (the tensors rlca_ppo_loss_fwd_bwd_weighted gets, after the same forward) into row `epoch`."""
        p = self.policy
        _lib.check(p.lib.rlca_ppo_diag_accumulate(p._workspace(nb), _ptr(p.flat), _ptr(value), _ptr(mean), _ptr(action),
                                                  _ptr(old_logprob), _ptr(adv), _ptr(target), nb, clip_value,
                                                  self.bound, _ptr(self.acc[epoch]), p._stream()))

    def grads(self, epoch):
        """The gradient buffer as the last rlca_policy_backward left it into row `epoch`."""
        p = self.policy
        _lib.check(p.lib.rlca_grad_sumsq(p._workspace(1), _ptr(p.grad), _ptr(self.acc[epoch]), p._stream()))

    def read(self):
        """The rows as a (epochs, COLUMNS) numpy array: one D2H."""
        return self.acc.cpu().numpy()

    def metrics(self):
        m = metrics(self.read())
        m['epochs_run'] = self.epochs_run
        m['logstd'] = [float(x) for x in self.policy.views['logstd'].tolist()]
        return m
