"""The learner kernels against a float64 reference at the batch sizes training runs them at.

Several kernel choices inside rlca_policy_forward / rlca_policy_backward depend on the batch size nb: the split-K
count of the fc1 tensor-core GEMM (8 / 4 / 2 / 1 k-splits for nb <= 896 / <= 1792 / <= 3712 / above), the 32- or
64-row tiles of the fp32 GEMMs, the number of samples each persistent conv-tower CTA walks (forward: nb over the SMs;
backward: nb over SMs / 2 slots, or SMs - 16 while a gradient event is set), and the zero padding of K = nb in the
dW_fc1 GEMM.  These tests run every one of those branches and compare with a plain float64 evaluation of the same
network (functional PyTorch in float64 on the GPU, autograd for the gradients).

The test batches are decisive (tests/learner_ref.py, which also holds the float64 reference): fp32 rounding cannot flip
a ReLU mask or the PPO clip branch on them, so every gradient tensor, the conv towers included, is held to one tight
bound.

Each comparison prints `[ratio] <what>: r` (error / bound); run with -s to see them.  A test makes all of its
comparisons before it fails, so a failure reports every ratio."""
import ctypes as C
import gc
import math

import numpy as np
import pytest
import torch

from golden_inputs import synthetic_state_dict
from learner_ref import (CLIP, COEFF, VCOEF, Checks, check_forward, decisive_pool, layer_scale, maxabs, params64,
                         ref_forward, ref_losses)

pytestmark = pytest.mark.gpu

POOL = 4136                  # decisive samples kept; the largest batch of the sweeps (the 4136-robot rollout)
FWD_NB = [1, 128, 129, 896, 897, 1024, 1032, 1792, 1793, 3712, 3713, 4104, 4136]
STEP_NB = [1, 67, 129, 512, 1000, 1024, 1793]
MODES = {1: 'tc', 2: 'fc1tc', 0: 'fp32'}      # set_tensor_cores: all tensor cores / fc1 GEMMs only / CUDA cores


def fc1_splits(nb):
    """k-splits of the fc1 forward GEMM (rlca_policy_forward): grow while 2 towers x 2 N tiles x M tiles x splits < 120"""
    mtiles, s = (nb + 127) // 128, 1
    while s < 8 and mtiles * 4 * s < 120:
        s *= 2
    return s


class Batch:
    """The first nb rows of the pool as float32 device tensors, the layout the C ABI takes"""

    def __init__(self, pool, nb):
        cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.nb = nb
        self.obs = cu(pool['obs'][:nb].reshape(nb, 1536))
        self.gs, self.act = cu(pool['gs'][:nb]), cu(pool['act'][:nb])
        self.old_lp, self.adv, self.tgt = cu(pool['old_lp'][:nb]), cu(pool['adv'][:nb]), cu(pool['tgt'][:nb])


@pytest.fixture(scope='module')
def pool(built):
    p = decisive_pool(POOL)
    assert p['survival'] > 0.3, f'only {p["survival"]:.1%} of the candidates are decisive: the fixture is broken'
    assert 0.2 < p['clipped'].mean() < 0.8, 'the batch should mix clipped and unclipped PPO ratios'
    p['ref_steps'] = {}
    return p


def ref_step(pool, nb, sd=None):
    """float64 value, mean, the three losses and all 23 gradients of one PPO minibatch (the pool's first nb rows)"""
    key = (nb, sd is None)
    if sd is None and key in pool['ref_steps']:
        return pool['ref_steps'][key]
    P = params64(synthetic_state_dict() if sd is None else sd, grad=True)
    d64 = lambda k: torch.from_numpy(pool[k][:nb]).cuda().double()
    v, mean, _ = ref_forward(P, d64('obs'), d64('gs'))
    (pl, vl, ent), loss = ref_losses(P, v, mean, d64('act'), d64('old_lp'), d64('adv'), d64('tgt'))
    loss.backward()
    out = dict(v=v.detach(), mean=mean.detach(), losses=[float(pl.detach()), float(vl.detach()), float(ent.detach())],
               grads={k: p.grad for k, p in P.items()})
    if sd is None:
        pool['ref_steps'][key] = out
    return out


# ------------------------------------------------------------------------------------------------ our side
def make_policy(max_batch, mode=1, sd=None):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=max_batch)
    pol.set_tensor_cores(mode)
    pol.load_state_dict({k: torch.as_tensor(v) for k, v in (synthetic_state_dict() if sd is None else sd).items()})
    return pol


def run_step(pol, b, weight=1.0, obs=None):
    """forward, PPO loss (+ its gradient, scaled by `weight`) and backward through the C ABI on the policy's workspace;
    returns copies of value, mean, the logged losses and the flat gradient"""
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.model.net import _ptr
    nb, obs = b.nb, b.obs if obs is None else obs
    lib, ws, st = pol.lib, pol._workspace(nb), pol._stream()
    v, mean = torch.empty(nb, device='cuda'), torch.empty(nb, 2, device='cuda')
    losses = torch.zeros(3, device='cuda')
    _lib.check(lib.rlca_policy_forward(ws, _ptr(pol.flat), _ptr(obs), _ptr(b.gs), nb, _ptr(v), _ptr(mean), st))
    _lib.check(lib.rlca_ppo_loss_fwd_bwd_weighted(ws, _ptr(pol.flat), _ptr(v), _ptr(mean), _ptr(b.act), _ptr(b.old_lp),
                                                  _ptr(b.adv), _ptr(b.tgt), nb, CLIP, COEFF, VCOEF, weight,
                                                  _ptr(losses), st))
    _lib.check(lib.rlca_policy_backward(ws, _ptr(pol.flat), _ptr(obs), _ptr(b.gs), nb, _ptr(pol.grad), st))
    torch.cuda.synchronize()
    return v.clone(), mean.clone(), losses.clone(), pol.grad.clone()


def grad_views(pol, flat):
    from rl_collision_avoidance_b200.model.net import TENSORS
    return {name: flat[pol.offsets[i]:pol.offsets[i] + math.prod(shape)].view(shape)
            for i, (name, shape) in enumerate(TENSORS)}


def unaligned(x):
    """a copy of x whose data pointer is 4 bytes past a 16-byte boundary (a view at storage offset 1)"""
    buf = torch.zeros(x.numel() + 4, device=x.device)
    u = buf[1:1 + x.numel()].view(x.shape)
    u.copy_(x)
    assert u.data_ptr() % 16 == 4
    return u


def check_step(what, pol, got, ref, grad_tol=5e-5):
    check = Checks()
    v, mean, losses, flat = got
    check_forward(check, what, v, mean, ref['v'], ref['mean'])
    for i, name in enumerate(('policy', 'value', 'entropy')):
        r = ref['losses'][i]
        check(f'{what} {name} loss', abs(float(losses[i]) - r), 1e-5 * max(abs(r), 1e-2))
    views = grad_views(pol, flat)
    for name, r in ref['grads'].items():
        check(f'{what} grad {name}', maxabs(views[name].double() - r), grad_tol * layer_scale(ref['grads'], name))
    check.done()


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize('mode', list(MODES), ids=list(MODES.values()))
@pytest.mark.parametrize('nb', FWD_NB, ids=[f'nb{n}-split{fc1_splits(n)}' for n in FWD_NB])
def test_forward_sweep_vs_float64(pool, nb, mode):
    """value, mean and both towers' relu(conv2) features across the fc1 split-K bands, the fp32 GEMM tile heights and
    the persistent conv-tower loop (several samples per CTA above 132 rows)"""
    b = Batch(pool, nb)
    pol = make_policy(nb, mode)
    v, mean = pol.forward_values(b.obs, b.gs)
    feats = [pol.features(t, nb) for t in range(2)]
    torch.cuda.synchronize()
    tag = f'fwd nb={nb} {MODES[mode]}'
    check = Checks()
    check_forward(check, tag, v, mean, torch.from_numpy(pool['v'][:nb]).cuda(), torch.from_numpy(pool['mean'][:nb]).cuda())
    P = params64(synthetic_state_dict())
    x64 = b.obs.double().view(nb, 3, 512)
    with torch.no_grad():
        for t in range(2):
            err, scale = 0.0, 1.0
            for r0 in range(0, nb, 1024):
                _, _, f_ref = ref_forward(P, x64[r0:r0 + 1024], b.gs[r0:r0 + 1024].double())
                err = max(err, maxabs(feats[t][r0:r0 + 1024].double() - f_ref[t]))
                scale = max(scale, maxabs(f_ref[t]))
            check(f'{tag} features tower {t}', err, 4e-6 * scale)
    check.done()


@pytest.mark.parametrize('mode', [1, 0], ids=['tc', 'fp32'])
@pytest.mark.parametrize('nb', STEP_NB, ids=[f'nb{n}' for n in STEP_NB])
def test_minibatch_step_vs_float64_autograd(pool, nb, mode):
    """The three losses and all 23 gradient tensors of one PPO minibatch against float64 autograd.  67 rows: one
    conv-backward slot holds two samples; 1000: ragged K of dW_fc1; 1793: split-K 2 and the 64-row dX GEMM."""
    b = Batch(pool, nb)
    pol = make_policy(nb, mode)
    check_step(f'step nb={nb} {MODES[mode]}', pol, run_step(pol, b), ref_step(pool, nb))


def test_workspace_reuse_is_bit_identical(pool):
    """One workspace sized for the largest batch serves full minibatches, the ragged tail and the rollout in turn.
    Every call equals, bit for bit, the same call on a fresh workspace and a repeat of itself."""
    pol = make_policy(POOL, 1)
    seen = {}
    for nb in (4104, 1024, 37, 1024, 1000):
        b = Batch(pool, nb)
        first = run_step(pol, b)
        again = run_step(pol, b)
        fresh_pol = make_policy(nb, 1)
        fresh = run_step(fresh_pol, b)
        del fresh_pol
        for name, a, r, f in zip(('value', 'mean', 'losses', 'gradient'), first, again, fresh):
            assert torch.equal(a, r), f'nb={nb}: {name} differs on a repeat of the same call'
            assert torch.equal(a, f), f'nb={nb}: {name} differs from a fresh workspace'
            if nb in seen:
                assert torch.equal(a, seen[nb][name]), f'nb={nb}: {name} differs from the earlier call at this size'
        seen[nb] = dict(zip(('value', 'mean', 'losses', 'gradient'), first))
    gc.collect()


@pytest.mark.parametrize('change', ['adam_step', 'load_state_dict'])
def test_unaligned_forward_keeps_conv_image_fresh(pool, change):
    """With the tensor-core conv tower on, an obs that is not 16-byte aligned takes the CUDA-core conv kernels.  A
    weight change followed by such a forward must still leave the tensor-core conv weight image to be rebuilt: the
    next aligned forward has to use the new conv weights."""
    from rl_collision_avoidance_b200.model.net import Adam
    nb = 256
    b = Batch(pool, nb)
    pol = make_policy(nb, 1)
    pol.forward_values(b.obs, b.gs)                                   # 1. aligned forward: builds the conv image
    if change == 'adam_step':                                         # 2. the weights change
        gen = torch.Generator(device='cuda').manual_seed(5)
        for g in pol.grad_views.values():
            g.copy_(torch.randn(g.shape, device='cuda', generator=gen))
        Adam(pol.parameters(), lr=1e-3).step()
    else:
        sd = {k: v * np.float32(1.01) if '_fea_cv' in k else v for k, v in synthetic_state_dict().items()}
        pol.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    pol.forward_values(unaligned(b.obs), b.gs)                        # 3. unaligned forward: CUDA-core conv tower
    v, mean = pol.forward_values(b.obs, b.gs)                         # 4. aligned forward
    torch.cuda.synchronize()
    sd_new = {k: t.cpu().numpy() for k, t in pol.state_dict().items()}
    fresh = make_policy(nb, 1, sd_new)
    v_f, mean_f = fresh.forward_values(b.obs, b.gs)
    torch.cuda.synchronize()
    with torch.no_grad():
        v_ref, mean_ref, _ = ref_forward(params64(sd_new), b.obs.double().view(nb, 3, 512), b.gs.double())
    check = Checks()
    check_forward(check, f'aligned after unaligned ({change})', v, mean, v_ref, mean_ref)
    if not (torch.equal(v, v_f) and torch.equal(mean, mean_f)):
        check.failed.append(f'the aligned forward after an unaligned one differs from a fresh policy with the new weights '
                            f'(max |dv| {maxabs(v - v_f):.3e}, max |dmean| {maxabs(mean - mean_f):.3e}): stale conv weights')
    check.done()


@pytest.mark.parametrize('nb', [1, 300])
def test_unaligned_obs_fallback_vs_float64(pool, nb):
    """forward, loss and backward of the tensor-core mode through the CUDA-core conv kernels (obs not 16-byte
    aligned; they read it with scalar loads) against float64 autograd"""
    b = Batch(pool, nb)
    pol = make_policy(nb, 1)
    check_step(f'unaligned nb={nb}', pol, run_step(pol, b, obs=unaligned(b.obs)), ref_step(pool, nb))


def test_weighted_loss_scales_every_gradient(pool):
    """rlca_ppo_loss_fwd_bwd_weighted (ranks of a data-parallel run with different row counts): the logged losses do not
    depend on the weight, every gradient is weight x the weight-1 gradient, and dlogstd = weight x g - coeff x weight
    (g: the policy-loss part)."""
    nb = 512
    b = Batch(pool, nb)
    pol = make_policy(nb, 1)
    _, _, loss1, g1 = run_step(pol, b, 1.0)
    off = pol.offsets
    check = Checks()
    for w in (0.25, 1.7):
        _, _, loss_w, g_w = run_step(pol, b, w)
        assert torch.equal(loss_w, loss1), f'weight {w}: logged losses changed'
        if w == 0.25:          # a power of two scales every rounding step exactly
            assert torch.equal(g_w, g1 * 0.25), 'weight 0.25: gradient is not exactly 0.25 x the weight-1 gradient'
        views_w, views_1 = grad_views(pol, g_w), grad_views(pol, g1)
        for name in views_1:
            if name == 'logstd':
                continue
            r = views_1[name].double() * w
            # at weight 1.7 every scaled summand rounds differently (and the fc1 GEMMs split it into other tf32 hi / lo
            # parts), and the sums cancel: act_fc1.weight moved by 1.24e-6 and act_fea_cv1.weight by 1.3e-6 of their scale
            check(f'weight {w} grad {name}', maxabs(views_w[name].double() - r), 4e-6 * maxabs(r))
        g = g1[off[0]:off[0] + 2].double() + COEFF           # policy-loss part of dlogstd at weight 1
        expect = w * g - COEFF * w
        check(f'weight {w} dlogstd', maxabs(g_w[off[0]:off[0] + 2].double() - expect), 1e-6 * maxabs(expect))
    check.done()


def test_grad_event_path(pool, monkeypatch):
    """With a gradient event set, the backward runs on one stream and the tensor-core conv backward on SMs - 16 CTAs
    (58 slots per tower on 132 SMs).  Non-conv gradients equal the single-stream backward bit for bit; the conv-tower
    gradients only sum their partials in other groups.  Clearing the event restores the default path."""
    from rl_collision_avoidance_b200 import _lib
    nb = 1024
    b = Batch(pool, nb)
    monkeypatch.setenv('RLCA_BWD_STREAMS', '0')          # read when the workspace is created (at the first forward)
    single_pol = make_policy(nb, 1)
    single = run_step(single_pol, b)
    monkeypatch.delenv('RLCA_BWD_STREAMS')
    default_pol = make_policy(nb, 1)
    default = run_step(default_pol, b)
    pol = make_policy(nb, 1)
    ws = pol._workspace(nb)
    ev = torch.cuda.Event()
    ev.record()                                           # creates the underlying cudaEvent_t
    _lib.check(pol.lib.rlca_policy_set_grad_event(ws, C.c_void_p(ev.cuda_event)))
    with_event = run_step(pol, b)
    check_step(f'grad event nb={nb}', pol, with_event, ref_step(pool, nb))
    for a, r in zip(with_event[:3], single[:3]):
        assert torch.equal(a, r)
    g_ev, g_single = grad_views(pol, with_event[3]), grad_views(pol, single[3])
    check = Checks()
    for name in g_ev:
        if '_fea_cv' in name:
            # regrouping the partial sums moved act_fea_cv1.weight (2.6e-3, a sum of ~2.6e5 products that cancels) by
            # 4.6e-6 of its scale; its fp32 error against float64 is 1.8e-5 of its scale on either path
            check(f'grad event {name} vs one stream', maxabs(g_ev[name] - g_single[name]), 1e-5 * maxabs(g_single[name]))
        else:
            assert torch.equal(g_ev[name], g_single[name]), f'{name}: the gradient-event path changed a non-conv gradient'
    check.done()
    _lib.check(pol.lib.rlca_policy_set_grad_event(ws, None))
    cleared = run_step(pol, b)
    for a, r, s in zip(cleared, default, single):
        assert torch.equal(a, r) and torch.equal(a, s), 'clearing the gradient event did not restore the default path'


def gae_ref(r, v, lv, d, gamma, lam):
    """model/ppo.py generate_train_data as a sequential float64 recurrence"""
    T, N = r.shape
    vals = np.vstack([v, lv[None]]).astype(np.float64)
    nd = 1.0 - d.astype(np.float64)
    gae, tg = np.zeros(N), np.zeros((T, N))
    for t in range(T - 1, -1, -1):
        delta = r[t].astype(np.float64) + gamma * vals[t + 1] * nd[t] - vals[t]
        gae = delta + gamma * lam * nd[t] * gae
        tg[t] = gae + vals[t]
    return tg, tg - vals[:-1]


@pytest.mark.parametrize('N', [1, 33, 4104])
@pytest.mark.parametrize('T', [1, 7, 8, 9, 128, 129])
def test_gae_vs_float64_recurrence(built, T, N):
    """rlca_gae (chunked segmented scan over time) against the sequential recurrence: done flags at t = 0, at
    t = T - 1 and a column done at every step; targets and advantages within 1 float32 ulp of the rounded reference."""
    from rl_collision_avoidance_b200.model.ppo import generate_train_data
    rs = np.random.RandomState(T * 10000 + N)
    r = rs.uniform(-1, 1, (T, N)).astype(np.float32)
    v = rs.uniform(-5, 5, (T, N)).astype(np.float32)
    lv = rs.uniform(-5, 5, N).astype(np.float32)
    d = rs.rand(T, N) < 0.15
    d[0, ::3] = True
    d[T - 1, 1::3] = True
    if N > 2:
        d[:, 2] = True
    cu = lambda a: torch.from_numpy(a).cuda()
    tg, adv = generate_train_data(cu(r), 0.99, cu(v), cu(lv), cu(d), 0.95)
    # the C ABI takes gamma and lambda as float32
    tg_ref, adv_ref = gae_ref(r, v, lv, d, float(np.float32(0.99)), float(np.float32(0.95)))
    check = Checks()
    for name, got, ref in (('targets', tg, tg_ref), ('advantages', adv, adv_ref)):
        ref32 = ref.astype(np.float32)
        err = np.abs(got.cpu().numpy().astype(np.float64) - ref32) / np.spacing(np.abs(ref32))
        check(f'gae T={T} N={N} {name} (ulps)', float(err.max()), 1.0)
    check.done()


def test_advantage_normalisation_at_rollout_size(built):
    """(adv - mean) / std over a 128 x 4104 rollout against float64"""
    from rl_collision_avoidance_b200.model.ppo import normalize_advantages
    rs = np.random.RandomState(7)
    x = (rs.standard_normal((128, 4104)) * 3 + 1.5).astype(np.float32)
    got = normalize_advantages(torch.from_numpy(x).cuda()).cpu().numpy()
    x64 = x.astype(np.float64)
    ref = (x64 - x64.mean()) / x64.std()
    check = Checks()
    check('advantage normalisation 128x4104', float(np.abs(got - ref).max()), 1e-6)
    check.done()


def test_forward_at_65544_rows(pool):
    """The policy forward at the 65 544-robot size of the raycast sweep (more rows than a grid's y dimension takes):
    rows at both ends against float64, every output finite."""
    nb = 65544
    need = 20 << 30                   # the workspace is about 17 GB at this size
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f'needs about {need >> 30} GB of free device memory, {free / 2 ** 30:.1f} GB free')
    idx = torch.arange(nb) % POOL
    x = torch.from_numpy(pool['obs'].reshape(POOL, 1536)).cuda()[idx.cuda()]
    gs = torch.from_numpy(pool['gs']).cuda()[idx.cuda()]
    pol = make_policy(nb, 1)
    v, mean = pol.forward_values(x, gs)
    torch.cuda.synchronize()
    assert torch.isfinite(v).all() and torch.isfinite(mean).all()
    v_ref, mean_ref = torch.from_numpy(pool['v']).cuda()[idx.cuda()], torch.from_numpy(pool['mean']).cuda()[idx.cuda()]
    check = Checks()
    for r0, r1 in ((0, 512), (nb - 512, nb)):
        check_forward(check, f'fwd nb={nb} rows {r0}..{r1}', v[r0:r1], mean[r0:r1], v_ref[r0:r1], mean_ref[r0:r1])
    check.done()
    del pol, x, gs, v, mean
    gc.collect()
    torch.cuda.empty_cache()
