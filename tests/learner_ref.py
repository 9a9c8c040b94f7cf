"""Float64 reference of the learner (CNNPolicy forward, PPO losses) and the decisive batches the learner tests use.

Decisive batches: every sample keeps each ReLU pre-activation (conv1, conv2, fc1 and fc2 of both towers) at least
MARGIN x (that layer's max |z|) away from zero, and its PPO ratio MARGIN away from 1 +- CLIP.  fp32 rounding cannot flip
a ReLU mask or the clip branch on such a batch, so the kernels and the float64 reference apply the same masks and every
gradient tensor, the conv towers included, is held to one tight bound.

`Checks` collects error <= bound comparisons: each prints `[ratio] <what>: r` (error / bound; run pytest with -s to see
them), and done() fails with every one that missed."""
import math

import numpy as np
import torch
import torch.nn.functional as Fn

from golden_inputs import synthetic_state_dict

CLIP, COEFF, VCOEF = 0.1, 5e-4, 20.0
MARGIN = 1e-5                # relative ReLU / absolute PPO-ratio margin of a decisive sample


class Checks:
    """error <= bound comparisons of one test: each prints its ratio, and done() fails with every one that missed"""

    def __init__(self):
        self.failed = []

    def __call__(self, what, err, bound):
        ratio = err / bound if bound > 0 else (0.0 if err == 0 else math.inf)
        print(f'[ratio] {what}: {ratio:.4f}')
        if not err <= bound:
            self.failed.append(f'{what}: error {err:.3e} exceeds the bound {bound:.3e}')

    def done(self):
        assert not self.failed, '\n'.join(self.failed)


def maxabs(t):
    return float(t.abs().max()) if t.numel() else 0.0


def check_forward(check, what, v, mean, v_ref, mean_ref):
    """the policy's value and mean against float64: 2e-5 of the value scale, 1e-5 absolute for the mean (in (0, 1) and
    (-1, 1))"""
    vs = max(1.0, maxabs(v_ref))
    check(f'{what} value', maxabs(v.double() - v_ref), 2e-5 * vs)
    check(f'{what} mean', maxabs(mean.double() - mean_ref), 1e-5)


def layer_scale(grads, name):
    """max |gradient| of the layer a tensor belongs to (weight and bias).  A bias gradient is the plain sum over the
    batch of the layer's upstream gradient and can cancel far below the size of its terms (the actor2 bias: 2.4e-3 at
    1000 rows, from summands whose forward rounding alone moves it by 1.5e-7), so it is held to its layer's scale."""
    layer = name.rsplit('.', 1)[0]
    if not name.endswith('.bias'):
        return maxabs(grads[name])
    return max(maxabs(r) for k, r in grads.items() if k.rsplit('.', 1)[0] == layer)


# ------------------------------------------------------------------------------------------------ float64 reference
def params64(sd, dev='cuda', grad=False):
    return {k: torch.as_tensor(np.asarray(v), dtype=torch.float64, device=dev).clone().requires_grad_(grad)
            for k, v in sd.items()}


def ref_forward(P, x, gs, pre=None):
    """CNNPolicy forward (model/net.py): x (n, 3, 512), gs (n, 4) = goal | speed -> value (n,), mean (n, 2) and the
    relu(conv2) features of both towers (n, 4096 each).  `pre` (a list) receives (layer, pre-activation) of every ReLU."""
    feats, hidden = [], []
    for p in ('act', 'crt'):
        z1 = Fn.conv1d(x, P[p + '_fea_cv1.weight'], P[p + '_fea_cv1.bias'], 2, 1)
        z2 = Fn.conv1d(torch.relu(z1), P[p + '_fea_cv2.weight'], P[p + '_fea_cv2.bias'], 2, 1)
        f = torch.relu(z2).flatten(1)
        z3 = Fn.linear(f, P[p + '_fc1.weight'], P[p + '_fc1.bias'])
        z4 = Fn.linear(torch.cat((torch.relu(z3), gs), 1), P[p + '_fc2.weight'], P[p + '_fc2.bias'])
        if pre is not None:
            pre += [(p + '_cv1', z1), (p + '_cv2', z2), (p + '_fc1', z3), (p + '_fc2', z4)]
        feats.append(f)
        hidden.append(torch.relu(z4))
    mean = torch.cat((torch.sigmoid(Fn.linear(hidden[0], P['actor1.weight'], P['actor1.bias'])),
                      torch.tanh(Fn.linear(hidden[0], P['actor2.weight'], P['actor2.bias']))), 1)
    v = Fn.linear(hidden[1], P['critic.weight'], P['critic.bias'])[:, 0]
    return v, mean, feats


def ref_logprob(P, mean, act):
    ls = P['logstd']
    return (-(act - mean) ** 2 / (2 * torch.exp(2 * ls)) - 0.5 * math.log(2 * math.pi) - ls).sum(1)


def ref_losses(P, v, mean, act, old_lp, adv, tgt):
    """model/ppo.py's clipped surrogate, value MSE and entropy; returns (policy, value, entropy) and the total loss"""
    ratio = torch.exp(ref_logprob(P, mean, act) - old_lp)
    pl = -torch.min(ratio * adv, torch.clamp(ratio, 1 - CLIP, 1 + CLIP) * adv).mean()
    vl = ((v - tgt) ** 2).mean()
    ent = (0.5 + 0.5 * math.log(2 * math.pi) + P['logstd']).sum()
    return (pl, vl, ent), pl + VCOEF * vl - COEFF * ent


# ------------------------------------------------------------------------------------------------ decisive batches
def candidate_batch(rs, n):
    """Scans like the env's: values in [-0.5, 0.5] in runs of equal values, about a third of the beams saturated at
    exactly +0.5 (free space), three frames that differ by a little noise per run; goal, speed and action in the
    ranges of golden_inputs.synthetic_batch; PPO advantages, value targets and a log-ratio offset."""
    run = np.cumsum(rs.rand(n, 512) < 0.2, axis=1)                       # run index of each beam, mean length 5
    level = rs.uniform(-0.5, 0.5, (n, 513))
    free = rs.rand(n, 513) < 1 / 3
    rows = np.arange(n)[:, None]
    base = level[rows, run]
    noise = 0.02 * rs.standard_normal((n, 3, 513))
    noise[:, 2] = 0.0                                                    # the newest frame is the base scan
    x = np.clip(base[:, None, :] + noise[rows[:, :, None], np.arange(3)[None, :, None], run[:, None, :]], -0.5, 0.5)
    x = np.where(free[rows, run][:, None, :], 0.5, x).astype(np.float32)
    goal = rs.uniform(-8, 8, (n, 2))
    speed = np.stack([rs.uniform(0, 1, n), rs.uniform(-1, 1, n)], 1)
    act = np.stack([rs.uniform(-0.2, 1.2, n), rs.uniform(-1.2, 1.2, n)], 1)
    return dict(obs=x, gs=np.concatenate([goal, speed], 1).astype(np.float32), act=act.astype(np.float32),
                adv=rs.standard_normal(n).astype(np.float32), tgt=rs.uniform(-3, 3, n).astype(np.float32),
                logratio=rs.uniform(-0.25, 0.25, n))


def decisive_pool(n, dev='cuda', seed=2024, chunk=2048):
    """The first n candidates whose ReLU pre-activations and PPO ratio are all decisive (module docstring), with their
    float64 value and mean.  old_lp is set so that the ratio of the float64 policy is exp(logratio), a mix of clipped
    and unclipped samples."""
    rs = np.random.RandomState(seed)
    P = params64(synthetic_state_dict(), dev)
    kept, seen = [], 0
    while sum(len(k['adv']) for k in kept) < n:
        c = candidate_batch(rs, chunk)
        seen += chunk
        x = torch.from_numpy(c['obs']).to(dev, torch.float64)
        gs = torch.from_numpy(c['gs']).to(dev, torch.float64)
        pre = []
        with torch.no_grad():
            v, mean, _ = ref_forward(P, x, gs, pre)
            ok = torch.ones(chunk, dtype=torch.bool, device=dev)
            for _, z in pre:
                delta = MARGIN * float(z.abs().max())
                ok &= (z.abs() >= delta).flatten(1).all(1)
            lp = ref_logprob(P, mean, torch.from_numpy(c['act']).to(dev, torch.float64))
            old_lp = (lp - torch.from_numpy(c['logratio']).to(dev)).float()
            ratio = torch.exp(lp - old_lp.double())
            ok &= ((ratio - (1 - CLIP)).abs() >= MARGIN) & ((ratio - (1 + CLIP)).abs() >= MARGIN)
        sel = ok.cpu().numpy()
        d = {k: c[k][sel] for k in ('obs', 'gs', 'act', 'adv', 'tgt')}
        d.update(old_lp=old_lp.cpu().numpy()[sel], v=v.cpu().numpy()[sel], mean=mean.cpu().numpy()[sel],
                 clipped=((ratio < 1 - CLIP) | (ratio > 1 + CLIP)).cpu().numpy()[sel])
        kept.append(d)
    pool = {k: np.concatenate([d[k] for d in kept])[:n] for k in kept[0]}
    first = int(np.argmin(pool['clipped']))         # an unclipped sample first: at nb = 1 every gradient is non-zero
    for k in pool:
        pool[k][[0, first]] = pool[k][[first, 0]]
    pool['survival'] = sum(len(d['adv']) for d in kept) / seen
    return pool
