"""PPO update diagnostics on the GPU (DESIGN.md §9n): rlca_ppo_diag_accumulate and rlca_grad_sumsq against the float64
reference of tests/diag_ref.py, the ratio against the loss kernel's own, the PPO update with the diagnostics off and
on bit for bit, the target-KL stop, and trainer.run with diagnostics."""
import ctypes as C

import numpy as np
import pytest
import torch

import diag_ref
from diag_ref import BOUND, CLIP, LOGSTD

pytestmark = pytest.mark.gpu

SIZES = (1, 31, 512, 1000, 1024, 4136)
ULP = float(np.finfo(np.float32).eps)


def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope='module')
def pol(built):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    p = CNNPolicy(seed=2, max_batch=max(SIZES))
    p.views['logstd'].copy_(torch.tensor(LOGSTD))
    return p


def new_diag(pol, epochs=1):
    from rl_collision_avoidance_b200.model.diagnostics import PPODiagnostics
    return PPODiagnostics(pol, epochs, [list(BOUND[0]), list(BOUND[1])])


def accumulate(diag, epoch, b):
    t = {k: cu(v) for k, v in b.items()}
    diag.accumulate(epoch, t['value'], t['mean'], t['action'], t['old_lp'], t['adv'], t['target'], len(b['adv']), CLIP)


def check_row(got, b):
    """One accumulator row against the float64 reference of the rows b: counts exact, sums to 1e-5 of their scale, the
    ratio extremes to a few ulp of the fp32 ratio."""
    from rl_collision_avoidance_b200.model.diagnostics import COL
    cols, scales = diag_ref.ref_row(b)
    for name in diag_ref.SUM_COLUMNS:
        if name in diag_ref.COUNT_COLUMNS:
            assert got[COL[name]] == cols[name], name
        else:
            assert abs(got[COL[name]] - cols[name]) <= 1e-5 * scales[name], (name, got[COL[name]], cols[name])
    r32 = diag_ref.ratio32(LOGSTD, b['mean'], b['action'], b['old_lp']).astype(np.float64)
    assert abs(got[COL['max_ratio']] - r32.max()) <= 8 * ULP * r32.max()
    assert abs(got[COL['min_ratio']] - r32.min()) <= 8 * ULP * r32.min()


@pytest.mark.parametrize('nb', SIZES)
def test_accumulate_matches_the_reference(pol, nb):
    from rl_collision_avoidance_b200.model.diagnostics import COL, EMPTY_ROW
    b = diag_ref.decisive_batch(np.random.RandomState(100 + nb), nb)
    diag = new_diag(pol)
    accumulate(diag, 0, b)
    got = diag.read()[0]
    check_row(got, b)
    g0 = COL['grad_steps']
    assert np.array_equal(got[g0:], EMPTY_ROW[g0:])                 # the gradient columns are rlca_grad_sumsq's
    if nb >= 512:                                                   # every count is exercised
        for name in diag_ref.COUNT_COLUMNS:
            assert 0 < got[COL[name]] < nb or name == 'n', name


def loss_of(pol, b):
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.model.net import _ptr
    nb = len(b['adv'])
    t = {k: cu(v) for k, v in b.items()}
    losses = torch.zeros(3, device='cuda')
    _lib.check(pol.lib.rlca_ppo_loss_fwd_bwd(pol._workspace(nb), _ptr(pol.flat), _ptr(t['value']), _ptr(t['mean']),
                                             _ptr(t['action']), _ptr(t['old_lp']), _ptr(t['adv']), _ptr(t['target']),
                                             nb, CLIP, 5e-4, 20.0, _ptr(losses), pol._stream()))
    return losses.cpu().numpy()


def test_ratio_is_the_loss_kernels(pol):
    """With A = 1 and every ratio inside the clip range the policy loss is -mean(r).  One row at a time it is -r, the
    loss kernel's fp32 ratio itself: the diagnostics must hold the same bits.  Over a batch the accumulated sum
    reproduces the loss."""
    from rl_collision_avoidance_b200.model.diagnostics import COL
    b = diag_ref.decisive_batch(np.random.RandomState(7), 600, spread=0.09)
    b['adv'][:] = 1.0
    for i in range(12):
        one = {k: v[i:i + 1] for k, v in b.items()}
        diag = new_diag(pol)
        accumulate(diag, 0, one)
        got = diag.read()[0]
        r = np.float32(-loss_of(pol, one)[0])
        assert got[COL['max_ratio']] == float(r) == got[COL['min_ratio']] == got[COL['sum_ratio']]
    b = {k: v[:256] for k, v in b.items()}
    diag = new_diag(pol)
    accumulate(diag, 0, b)
    got = diag.read()[0]
    assert got[COL['clipped']] == 0 and got[COL['cut']] == 0
    assert abs(-got[COL['sum_ratio']] / got[COL['n']] - float(loss_of(pol, b)[0])) < 1e-6


def test_deterministic_additive_and_per_epoch(pol):
    rs = np.random.RandomState(9)
    b1, b2, b3 = (diag_ref.decisive_batch(rs, n) for n in (700, 333, 64))
    runs = []
    for _ in range(2):
        diag = new_diag(pol, epochs=3)
        accumulate(diag, 0, b1)
        accumulate(diag, 2, b3)
        accumulate(diag, 0, b2)
        runs.append(diag.read())
    assert np.array_equal(runs[0].view(np.uint64), runs[1].view(np.uint64))        # the same bits
    from rl_collision_avoidance_b200.model.diagnostics import EMPTY_ROW
    check_row(runs[0][0], diag_ref.union([b1, b2]))
    assert np.array_equal(runs[0][1], EMPTY_ROW)
    check_row(runs[0][2], b3)


def test_bad_arguments_are_errors(pol):
    from rl_collision_avoidance_b200 import _lib
    diag = new_diag(pol)
    b = diag_ref.decisive_batch(np.random.RandomState(1), 8)
    t = {k: cu(v) for k, v in b.items()}
    ptr = lambda x: C.c_void_p(x.data_ptr())
    for nb in (0, -3, pol._ws_batch + 1):
        with pytest.raises(_lib.RlcaError, match='max_batch'):
            _lib.check(pol.lib.rlca_ppo_diag_accumulate(pol._workspace(1), ptr(pol.flat), ptr(t['value']), ptr(t['mean']),
                                                        ptr(t['action']), ptr(t['old_lp']), ptr(t['adv']),
                                                        ptr(t['target']), nb, CLIP, diag.bound, ptr(diag.acc),
                                                        pol._stream()))
    with pytest.raises(_lib.RlcaError, match='NULL'):
        diag.accumulate(0, t['value'], None, t['action'], t['old_lp'], t['adv'], t['target'], 8, CLIP)
    with pytest.raises(_lib.RlcaError, match='NULL'):
        _lib.check(pol.lib.rlca_grad_sumsq(pol._workspace(1), None, C.c_void_p(diag.acc.data_ptr()), pol._stream()))


def test_grad_sumsq_matches_float64(pol):
    """On the gradient of a real backward: per tensor and in total, with the padding between the tensors poisoned (it
    must not be read), twice into one row (sums add, the step count goes up, the max column keeps the larger call)."""
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.model.diagnostics import COL, EMPTY_ROW
    from rl_collision_avoidance_b200.model.net import TENSORS, _ptr
    nb = 256
    rs = np.random.RandomState(3)
    b = diag_ref.decisive_batch(rs, nb)
    obs = cu((rs.rand(nb, 3, 512) - 0.5).astype(np.float32))
    gs = cu(rs.uniform(-1, 1, (nb, 4)).astype(np.float32))
    v, mean = pol.forward_values(obs, gs)
    losses = torch.zeros(3, device='cuda')
    ws, st = pol._workspace(nb), pol._stream()
    _lib.check(pol.lib.rlca_ppo_loss_fwd_bwd(ws, _ptr(pol.flat), _ptr(v), _ptr(mean), _ptr(cu(b['action'])),
                                             _ptr(cu(b['old_lp'])), _ptr(cu(b['adv'])), _ptr(cu(b['target'])), nb, CLIP,
                                             5e-4, 20.0, _ptr(losses), st))
    _lib.check(pol.lib.rlca_policy_backward(ws, _ptr(pol.flat), _ptr(obs), _ptr(gs), nb, _ptr(pol.grad), st))
    sizes = [int(np.prod(shape)) for _, shape in TENSORS]
    offsets = pol.offsets[:-1]
    inside = torch.zeros(pol.flat_size, dtype=torch.bool, device='cuda')
    for o, n in zip(offsets, sizes):
        inside[o:o + n] = True
    assert int((~inside).sum()) > 0
    g1 = torch.where(inside, pol.grad, torch.full_like(pol.grad, 1e3))
    g2 = torch.where(inside, 0.5 * pol.grad, torch.full_like(pol.grad, -7.0))
    ref1 = diag_ref.ref_grad_sumsq(g1.cpu().numpy(), offsets, sizes)
    ref2 = diag_ref.ref_grad_sumsq(g2.cpu().numpy(), offsets, sizes)
    assert (ref1 > 0).all()                                         # every tensor has a gradient
    diag = new_diag(pol, epochs=2)
    row = C.c_void_p(diag.acc[1].data_ptr())
    for g in (g1, g2):
        _lib.check(pol.lib.rlca_grad_sumsq(ws, _ptr(g), row, st))
    got = diag.read()
    assert np.array_equal(got[0], EMPTY_ROW)
    k0 = COL['grad_sumsq.logstd']
    assert np.allclose(got[1][k0:k0 + 23], ref1 + ref2, rtol=1e-12, atol=0)
    assert got[1][COL['grad_steps']] == 2
    assert got[1][COL['max_grad_sumsq']] == pytest.approx(ref1.sum(), rel=1e-12)
    assert np.array_equal(got[1][:COL['grad_steps']], EMPTY_ROW[:COL['grad_steps']])
    for g in (g1, g2):                                              # and the same bits again
        _lib.check(pol.lib.rlca_grad_sumsq(ws, _ptr(g), C.c_void_p(diag.acc[0].data_ptr()), st))
    again = diag.read()
    assert np.array_equal(again[0].view(np.uint64), got[1].view(np.uint64))
    diag.acc[0].copy_(torch.from_numpy(EMPTY_ROW))
    diag.grads(0)                                                   # the method reads policy.grad
    m = diag.read()[0]
    assert m[COL['max_grad_sumsq']] == pytest.approx(ref1.sum(), rel=1e-12)


# ------------------------------------------------------------------------------------------------ the PPO update
T, N, BS, EPOCHS = 8, 40, 128, 3


def rollout(seed=4):
    """A rollout the policy itself sampled: (policy, memory, dones)."""
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    from rl_collision_avoidance_b200.model.ppo import generate_train_data
    rs = np.random.RandomState(seed)
    pol = CNNPolicy(seed=seed, max_batch=T * N)
    n = T * N
    level = rs.uniform(-0.5, 0.5, (n, 1, 512))
    obs = cu(np.clip(level + 0.05 * rs.standard_normal((n, 3, 512)), -0.5, 0.5).astype(np.float32))
    goal = cu(rs.uniform(-8, 8, (n, 2)).astype(np.float32))
    speed = cu(np.stack([rs.uniform(0, 1, n), rs.uniform(-1, 1, n)], 1).astype(np.float32))
    v, a, lp, _ = pol.forward(obs, goal, speed)
    rewards = cu(rs.uniform(-1, 1, (T, N)).astype(np.float32))
    dones = rs.rand(T, N) < 0.3
    last_v = cu(rs.uniform(-1, 1, N).astype(np.float32))
    values = v.reshape(T, N).clone()
    tg, adv = generate_train_data(rewards, 0.99, values, last_v, cu(dones), 0.95)
    memory = (obs.reshape(T, N, 3, 512), goal.reshape(T, N, 2), speed.reshape(T, N, 2), a.reshape(T, N, 2).clone(),
              lp.reshape(T, N).clone(), tg, values, rewards, adv)
    return pol, memory, dones


def run_update(stage, diagnostics, target_kl=None, epochs=EPOCHS, bs=BS, lr=5e-5):
    """One update from the same start on recorded permutations: (loss rows, parameters, both moments, steps, diag)."""
    from rl_collision_avoidance_b200.model.net import Adam
    from rl_collision_avoidance_b200.model.ppo import ppo_update_stage1, ppo_update_stage2
    from rl_collision_avoidance_b200.model.utils import get_filter_index
    pol, memory, dones = rollout()
    opt = Adam(pol.parameters(), lr=lr)
    diag = new_diag(pol, epochs) if diagnostics else None
    kw = dict(batch_size=bs, memory=memory, epoch=epochs, coeff_entropy=5e-4, clip_value=CLIP, num_step=T, num_env=N,
              frames=3, obs_size=512, act_size=2, diagnostics=diag, target_kl=target_kl)
    rs = np.random.RandomState(77)
    if stage == 1:
        rows = ppo_update_stage1(pol, opt, permutations=[rs.permutation(T * N) for _ in range(epochs)], **kw)
    else:
        filt = get_filter_index(dones)
        assert 0 < len(filt) < T * N
        kept = T * N - len(filt)
        rows = ppo_update_stage2(pol, opt, filter_index=filt, permutations=[rs.permutation(kept) for _ in range(epochs)], **kw)
    torch.cuda.synchronize()
    return rows, pol.flat.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.step_count, diag


def same_bits(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a[1:4], b[1:4])) and a[0] == b[0] \
        and a[4] == b[4]


@pytest.mark.parametrize('stage', [1, 2])
def test_update_is_the_same_with_diagnostics(built, stage):
    off = run_update(stage, False)
    on = run_update(stage, True)
    assert len(off[0]) == off[4] > EPOCHS and same_bits(off, on)
    diag = on[5]
    m = diag.metrics()
    assert m['epochs_run'] == EPOCHS and len(m['per_epoch']) == EPOCHS
    steps = off[4] // EPOCHS
    acc = diag.read()
    from rl_collision_avoidance_b200.model.diagnostics import COL
    assert (acc[:, COL['grad_steps']] == steps).all()
    rows_per_epoch = T * N if stage == 1 else steps * BS
    assert (acc[:, COL['n']] == rows_per_epoch).all()
    kl = [e['approx_kl_k3'] for e in m['per_epoch']]
    assert 0 < kl[0] < kl[1] < kl[2]                                # every epoch moves the policy further
    assert all(np.isfinite(e['grad_norm']) and e['grad_norm'] > 0 for e in m['per_epoch'])
    assert m['grad_norm_max'] >= m['grad_norm'] and m['logstd'] == diag.policy.views['logstd'].tolist()


def test_policy_has_not_moved_in_the_first_minibatch(built):
    """One epoch of one minibatch over the whole rollout: the parameters are the ones that sampled it."""
    res = run_update(1, True, epochs=1, bs=T * N)
    m = res[5].metrics()
    assert res[4] == 1 and m['rows'] == T * N
    assert abs(m['approx_kl']) < 1e-5 and abs(m['approx_kl_k3']) < 1e-5
    assert abs(m['ratio_max'] - 1) < 1e-4 and abs(m['ratio_min'] - 1) < 1e-4 and m['clip_fraction'] == 0
    assert 0 <= m['action_saturation'][0] <= 1 and m['mean_saturation'] == [0.0, 0.0]


@pytest.mark.parametrize('stage', [1, 2])
def test_target_kl_stops_the_epochs(built, stage):
    free = run_update(stage, True)
    steps = free[4] // EPOCHS
    tiny = run_update(stage, True, target_kl=1e-9)
    assert tiny[5].epochs_run == 1 and tiny[4] == steps == len(tiny[0])
    assert tiny[0] == free[0][:steps]
    m = tiny[5].metrics()
    assert m['epochs_run'] == 1 and [e['rows'] > 0 for e in m['per_epoch']] == [True, False, False]
    huge = run_update(stage, True, target_kl=1e9)
    assert huge[5].epochs_run == EPOCHS and same_bits(free, huge)
    kl0, kl1 = (e['approx_kl_k3'] for e in free[5].metrics()['per_epoch'][:2])
    assert 1e-9 < kl0 < kl1
    mid = run_update(stage, True, target_kl=0.5 * (kl0 + kl1))       # stops after epoch 1, not after epoch 0
    assert mid[5].epochs_run == 2 and mid[4] == 2 * steps
    with pytest.raises(ValueError, match='target_kl needs diagnostics'):
        run_update(stage, False, target_kl=0.01)


def test_trainer_reports_diagnostics(built, tmp_path):
    import logging
    import socket
    from rl_collision_avoidance_b200.model import diagnostics as D
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.stage_world1 import StageWorld
    from rl_collision_avoidance_b200.trainer import run
    env = StageWorld(512, index=0, num_env=24, num_worlds=2, seed=1, auto_reset=1)
    policy = CNNPolicy(frames=3, action_space=2, seed=1, max_batch=max(256, env.N))
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=32, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=256, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=24, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    assert not D.logger_diag.handlers
    D.setup_diag_log(str(tmp_path))
    try:
        stats = run(env=env, policy=policy, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp,
                    stage=1, max_updates=2, diagnostics=True)
    finally:
        for h in list(D.logger_diag.handlers):
            h.close()
            D.logger_diag.removeHandler(h)
    assert len(stats) == 2
    for s in stats:
        m = s['diagnostics']
        assert m['epochs_run'] == 2 and m['rows'] == 2 * 32 * env.N
        scalars = [m[k] for k in ('approx_kl', 'approx_kl_k3', 'clip_fraction', 'cut_fraction', 'ratio_mean',
                                  'ratio_max', 'ratio_min', 'explained_variance', 'value_rmse', 'value_bias',
                                  'adv_mean', 'adv_std', 'grad_norm', 'grad_norm_max')]
        scalars += m['mean_saturation'] + m['action_saturation'] + m['logstd'] + list(m['grad_norm_by_group'].values())
        assert np.isfinite(scalars).all(), m
        assert 0 <= m['cut_fraction'] <= m['clip_fraction'] <= 1
        assert m['ratio_min'] <= m['ratio_mean'] <= m['ratio_max']
        assert abs(m['adv_mean']) < 1e-3 and abs(m['adv_std'] - 1) < 1e-3           # normalised over the rollout
        e0, e1 = m['per_epoch']
        # the k3 estimator is never negative and has far less noise than old_lp - new_lp, whose mean over one epoch
        # of a 5e-5 step is smaller than its own sampling error
        assert e0['approx_kl_k3'] < e1['approx_kl_k3'] and e1['approx_kl_k3'] > 0
    lines = open(tmp_path / socket.gethostname() / 'diag.log').read().splitlines()
    assert len(lines) == 2 and lines[0].startswith('update 1, epochs 2, ') and lines[1].startswith('update 2, ')
    # off by default: the stats carry no diagnostics
    plain = run(env=env, policy=policy, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp, stage=1,
                max_updates=1)
    assert 'diagnostics' not in plain[0]
