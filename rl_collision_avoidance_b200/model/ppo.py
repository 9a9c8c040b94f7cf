"""PPO functions over device tensors (mirror of /root/reference/model/ppo.py:22-259).

Same names and argument order; numpy arrays become device tensors and every heavy step is a
librlca.so kernel: GAE (float64 recurrence), advantage normalisation, minibatch gather, policy
forward, fused clipped-surrogate/value/entropy loss + gradient, backward, fused Adam.
`ppo.log` gets the same "policy_loss, value_loss, entropy" line per minibatch (model/ppo.py:189-192),
written once per update from a device-side log instead of three host syncs per minibatch.
"""
from __future__ import annotations

import ctypes as C
import logging
import os
import socket

import torch

from .. import _lib
from .net import CNNPolicy, _ptr

logger_ppo = logging.getLogger('loggerppo')


def setup_ppo_log(root='./log'):
    """The reference creates ./log/<hostname>/ppo.log at import (model/ppo.py:10-19); here it is explicit."""
    d = os.path.join(root, socket.gethostname())
    os.makedirs(d, exist_ok=True)
    logger_ppo.setLevel(logging.INFO)
    if not logger_ppo.handlers:
        h = logging.FileHandler(os.path.join(d, 'ppo.log'), mode='a')
        h.setLevel(logging.INFO)
        logger_ppo.addHandler(h)
    return logger_ppo


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def transform_buffer(buff):
    """list of (state_list, a, r, d, logprob, v) per step -> 8 stacked tensors (model/ppo.py:22-54).
    state_list is (obs_stack (N,3,B), goal (N,2), speed (N,2))."""
    s_batch = torch.stack([e[0][0] for e in buff])
    goal_batch = torch.stack([e[0][1] for e in buff])
    speed_batch = torch.stack([e[0][2] for e in buff])
    a_batch = torch.stack([e[1] for e in buff])
    r_batch = torch.stack([e[2] for e in buff])
    d_batch = torch.stack([e[3] for e in buff])
    l_batch = torch.stack([e[4] for e in buff])
    v_batch = torch.stack([e[5] for e in buff])
    return s_batch, goal_batch, speed_batch, a_batch, r_batch, d_batch, l_batch, v_batch


def generate_action(env, state_list, policy, action_bound, out=None):
    """(v, a, logprob, scaled_action) for the whole batch (model/ppo.py:57-82).  env.index is always 0.
    state_list = (obs_stack (N,3,B), goal (N,2), speed (N,2)) or (obs_stack, gs (N,4)).  The clip to
    action_bound [[0,-1],[1,1]] happens in the sampling kernel; `out` may hold rollout slices."""
    assert list(map(float, action_bound[0])) == [0.0, -1.0] and list(map(float, action_bound[1])) == [1.0, 1.0], \
        'the sampling kernel clips to the reference action bound (ppo_stage1.py:170)'
    out = dict(out or {})
    if 'scaled' not in out:
        out['scaled'] = torch.empty(state_list[0].shape[0], 2, device=policy.device)
    if len(state_list) == 2:
        v, a, logprob, mean = policy.forward(state_list[0], None, None, gs=state_list[1], out=out)
    else:
        v, a, logprob, mean = policy.forward(state_list[0], state_list[1], state_list[2], out=out)
    return v, a, logprob, out['scaled']


def generate_action_no_sampling(env, state_list, policy, action_bound):
    """(mean, scaled_action) (model/ppo.py:84-107)"""
    obs, goal, speed = state_list
    _, mean = policy.forward_values(obs.contiguous(), policy._pack_gs(goal, speed))
    lo = torch.as_tensor(action_bound[0], device=mean.device, dtype=mean.dtype)
    hi = torch.as_tensor(action_bound[1], device=mean.device, dtype=mean.dtype)
    return mean, torch.minimum(torch.maximum(mean, lo), hi)


def generate_train_data(rewards, gamma, values, last_value, dones, lam):
    """GAE targets and advantages (model/ppo.py:122-139); (T,N) device tensors in, fp32 out."""
    lib = _lib.load()
    T, N = rewards.shape[0], rewards.shape[1]
    dev = rewards.device
    r = rewards.reshape(T, N).float().contiguous()
    v = values.reshape(T, N).float().contiguous()
    lv = last_value.reshape(N).float().contiguous()
    d = dones.reshape(T, N).to(torch.uint8).contiguous()
    targets = torch.empty(T, N, device=dev)
    advs = torch.empty(T, N, device=dev)
    _lib.check(lib.rlca_gae(_ptr(r), _ptr(v), _ptr(lv), _ptr(d), T, N, gamma, lam, _ptr(targets), _ptr(advs),
                            _stream(dev)))
    return targets, advs


def normalize_advantages(advs, process_group=None):
    """advs = (advs - advs.mean()) / advs.std() over the WHOLE rollout (model/ppo.py:148).  With a
    process group the three moments are all-reduced so every rank normalises with the global statistics
    (SURVEY.md §8(e))."""
    lib = _lib.load()
    dev = advs.device
    x = advs.reshape(-1).float().contiguous()
    mom = torch.empty(3, dtype=torch.float64, device=dev)
    _lib.check(lib.rlca_adv_moments(_ptr(x), x.numel(), _ptr(mom), _stream(dev)))
    if process_group is not None:
        from ..parallel import allreduce_moments
        allreduce_moments(mom, None if process_group is True else process_group)
    out = torch.empty_like(x)
    _lib.check(lib.rlca_adv_apply(_ptr(x), x.numel(), _ptr(mom), _ptr(out), _stream(dev)))
    return out.view(advs.shape)


class _MinibatchGather:
    """The arrays of a minibatch gathered by one sampler index in ONE launch (rlca_gather_minibatch); the pointer
    tables are built once per update."""

    def __init__(self, lib, srcs, dsts, rows, dev):
        import ctypes as C
        self.lib, self.n, self.dev = lib, len(srcs), dev
        self.keep = (srcs, dsts)                                  # the tensors whose addresses the tables hold
        self.src = (C.c_void_p * self.n)(*[t.data_ptr() for t in srcs])
        self.dst = (C.c_void_p * self.n)(*[t.data_ptr() for t in dsts])
        self.rows = (C.c_int32 * self.n)(*rows)

    def __call__(self, index):
        _lib.check(self.lib.rlca_gather_minibatch(self.src, self.rows, self.n, _ptr(index), index.numel(), self.dst,
                                                  _stream(self.dev)))


def _ppo_update(policy: CNNPolicy, optimizer, batch_size, memory, epoch, coeff_entropy, clip_value, num_step, num_env,
                frames, obs_size, act_size, filter_index=None, drop_last=False, generator=None, process_group=None,
                value_coef=20.0, permutations=None, diagnostics=None, target_kl=None):
    """Body shared by ppo_update_stage1/2.  `permutations` (optional, one index array per epoch into the KEPT rows)
    replays a recorded SubsetRandomSampler order instead of drawing one (parity tests against the reference).
    Under a process group the minibatch schedule is agreed across ranks first (parallel.plan_minibatches), so ranks
    with different row counts issue the same number of all-reduces.
    `diagnostics` (a diagnostics.PPODiagnostics, DESIGN.md §9n) accumulates every minibatch and its local gradient into
    the row of its epoch; losses, weights and ppo.log are the same with and without it.  With `target_kl` the finished
    epoch's row is read at every epoch boundary - one synchronisation each - and the remaining epochs are skipped once
    its approx_kl_k3 exceeds target_kl; under a process group the row is merged over the ranks first, so all of them
    stop together.  diagnostics.epochs_run is the number of epochs run."""
    if target_kl is not None and diagnostics is None:
        raise ValueError('target_kl needs diagnostics: the stop rule reads their rows')
    if diagnostics is not None and diagnostics.epochs < epoch:
        raise ValueError('the diagnostics hold %d epochs, the update runs %d' % (diagnostics.epochs, epoch))
    lib = _lib.load()
    obss, goals, speeds, actions, logprobs, targets, values, rewards, advs = memory
    dev = policy.device
    advs = normalize_advantages(advs, process_group)
    n_all = num_step * num_env
    obss = obss.reshape(n_all, frames * obs_size).float().contiguous()
    gs = torch.cat((goals.reshape(n_all, 2), speeds.reshape(n_all, 2)), dim=1).float().contiguous()
    actions = actions.reshape(n_all, act_size).float().contiguous()
    logprobs = logprobs.reshape(n_all).float().contiguous()
    advs = advs.reshape(n_all).float().contiguous()
    targets = targets.reshape(n_all).float().contiguous()
    keep = torch.arange(n_all, device=dev)
    if filter_index is not None and len(filter_index) > 0:      # np.delete(..., filter_index, 0) (model/ppo.py:212-218)
        mask = torch.ones(n_all, dtype=torch.bool, device=dev)
        mask[torch.as_tensor(list(filter_index), device=dev, dtype=torch.long)] = False
        keep = keep[mask]
    n = keep.numel()
    world = 1
    group = None if process_group in (None, True) else process_group
    if process_group is not None:
        import torch.distributed as dist
        world = dist.get_world_size(group)
    from ..parallel import OverlappedGradSync, allreduce_diagnostics, average_gradients, plan_minibatches
    from .diagnostics import RULES, over_target_kl
    # gradient exchange of a data-parallel run, in order of preference: (1) optimizer.peer (parallel.PeerAdam): the sum
    # over the ranks is part of the fused Adam kernel, nothing to do here; (2) one NCCL all-reduce of the flat buffer
    # after the backward; (3) RLCA_DP_OVERLAP=1: the fc-side ranges all-reduced under the rest of the backward
    # (parallel.OverlappedGradSync - no gain measured at N = 2 with NCCL's default channel count, DESIGN.md §9)
    sync = None
    peer = getattr(optimizer, 'peer', None) is not None
    if process_group is not None and not peer and os.environ.get('RLCA_DP_OVERLAP', '0') == '1':
        sync = getattr(policy, '_grad_sync', None)
        if sync is None or sync.group is not group:
            sync = policy._grad_sync = OverlappedGradSync(policy, group)
    bs = batch_size
    nbatches, sizes, weights = plan_minibatches(n, bs, drop_last, group, distributed=process_group is not None)
    b_obs = torch.empty(bs, frames * obs_size, device=dev)
    b_gs = torch.empty(bs, 4, device=dev)
    b_act = torch.empty(bs, act_size, device=dev)
    b_lp = torch.empty(bs, device=dev)
    b_adv = torch.empty(bs, device=dev)
    b_tgt = torch.empty(bs, device=dev)
    v = torch.empty(bs, device=dev)
    mean = torch.empty(bs, 2, device=dev)
    log = torch.zeros(max(1, epoch * nbatches), 3, device=dev)
    ws = policy._workspace(bs)
    st = _stream(dev)
    gather = _MinibatchGather(lib, (obss, gs, actions, logprobs, advs, targets), (b_obs, b_gs, b_act, b_lp, b_adv, b_tgt),
                              (frames * obs_size, 4, act_size, 1, 1, 1), dev)
    k = 0
    if diagnostics is not None:
        diagnostics.reset()
    for update in range(epoch):
        if permutations is not None:
            perm = keep[torch.as_tensor(permutations[update], device=dev, dtype=torch.long)]
        else:
            perm = keep[torch.randperm(n, device=dev, generator=generator)]     # SubsetRandomSampler (model/ppo.py:159)
        for bi in range(nbatches):
            nb = sizes[bi]
            if nb > 0:
                index = perm[bi * bs:bi * bs + nb].contiguous()
                gather(index)
                _lib.check(lib.rlca_policy_forward(ws, _ptr(policy.flat), _ptr(b_obs), _ptr(b_gs), nb, _ptr(v), _ptr(mean), st))
                _lib.check(lib.rlca_ppo_loss_fwd_bwd_weighted(ws, _ptr(policy.flat), _ptr(v), _ptr(mean), _ptr(b_act),
                                                              _ptr(b_lp), _ptr(b_adv), _ptr(b_tgt), nb, clip_value,
                                                              coeff_entropy, value_coef, float(weights[bi]),
                                                              _ptr(log[k]), st))
                if diagnostics is not None:
                    diagnostics.accumulate(update, v, mean, b_act, b_lp, b_adv, b_tgt, nb, clip_value)
                _lib.check(lib.rlca_policy_backward(ws, _ptr(policy.flat), _ptr(b_obs), _ptr(b_gs), nb, _ptr(policy.grad), st))
                if diagnostics is not None:
                    diagnostics.grads(update)
            else:
                policy.grad.zero_()             # this rank ran out of rows: it still takes part in the all-reduce
                if sync is not None:
                    sync.mark_ready()
            if sync is not None:
                sync.reduce()                   # fc-side ranges overlap the dF GEMM + conv tower backward
            elif process_group is not None and not peer:
                average_gradients(policy.grad, group)
            optimizer.step(grad_scale=1.0 / world)
            k += 1
        if diagnostics is not None:
            diagnostics.epochs_run = update + 1
        if target_kl is not None and update + 1 < epoch:
            row = diagnostics.acc[update].clone()
            if process_group is not None:
                allreduce_diagnostics(row, RULES, group)
            if over_target_kl(row.cpu().numpy(), target_kl):
                break
    if diagnostics is not None and process_group is not None:
        allreduce_diagnostics(diagnostics.acc, RULES, group)    # every rank reports the update of all ranks
    rows = log[:k].cpu().tolist()
    for pl, vl, ent in rows:
        logger_ppo.info('{}, {}, {}'.format(pl, vl, ent))
    return rows


def ppo_update_stage1(policy, optimizer, batch_size, memory, epoch, coeff_entropy=0.02, clip_value=0.2, num_step=2048,
                      num_env=12, frames=1, obs_size=24, act_size=4, generator=None, process_group=None,
                      permutations=None, diagnostics=None, target_kl=None, filter_index=None):
    """model/ppo.py:143-194 (drop_last=False).  `filter_index` (flat rows t * num_env + i) leaves rows out of the
    update, as stage 2's does; None is the reference's update over every row."""
    rows = _ppo_update(policy, optimizer, batch_size, memory, epoch, coeff_entropy, clip_value, num_step, num_env,
                       frames, obs_size, act_size, filter_index, False, generator, process_group,
                       permutations=permutations, diagnostics=diagnostics, target_kl=target_kl)
    print('update')
    return rows


def ppo_update_stage2(policy, optimizer, batch_size, memory, filter_index, epoch, coeff_entropy=0.02, clip_value=0.2,
                      num_step=2048, num_env=12, frames=1, obs_size=24, act_size=4, generator=None, process_group=None,
                      permutations=None, diagnostics=None, target_kl=None):
    """model/ppo.py:197-259 (filtered transitions deleted, drop_last=True)."""
    rows = _ppo_update(policy, optimizer, batch_size, memory, epoch, coeff_entropy, clip_value, num_step, num_env,
                       frames, obs_size, act_size, filter_index, True, generator, process_group,
                       permutations=permutations, diagnostics=diagnostics, target_kl=target_kl)
    print('filter {} transitions; update'.format(len(filter_index)))
    return rows
