"""The data-parallel PPO update (model/ppo.py _ppo_update with a process group) with G processes on one GPU.

G ordinary processes share the device and a gloo process group (gloo all-reduces CUDA tensors through the host; NCCL
would refuse two ranks on one device).  Each rank builds CNNPolicy from golden_inputs.synthetic_state_dict() and takes
its own slice of a decisive batch pool (tests/learner_ref.py; decisive for clip 0.1 and entropy coefficient 5e-4), then
runs ppo_update_stage1 or ppo_update_stage2 on recorded permutations, so that the test knows which rows every rank used
in every optimizer step.  Stage 1 gives the ranks different row counts, so that one rank takes a short minibatch and
another an empty one; stage 2 deletes a different `filter_index` on every rank and drops the ranks' tails.  Every case
runs with the plain gradient all-reduce and with RLCA_DP_OVERLAP=1 (parallel.OverlappedGradSync: the fc-side ranges
all-reduced from a side stream while the backward still runs).

Checks:
  * with lr = 0 (every step sees the same parameters, the pool stays decisive) the gradient each rank hands to Adam,
    policy.grad x grad_scale, is the same bits on every rank and matches the float64 autograd gradient of the PPO loss
    over the union of all ranks' rows of that step, with the advantages normalised in float64 over the union of the
    ranks' rollouts (per layer, 5e-5 of the layer's gradient scale, as the single-rank learner tests);
  * normalize_advantages(advs, True) on each rank equals that float64 normalisation to 1e-6;
  * every rank takes the same number of optimizer steps, the number the minibatch schedule rule gives;
  * with lr = 5e-5 and two epochs every rank ends with the same bits of parameters and both Adam moments.

Each float64 comparison prints `[ratio] <what>: r` (error / bound); run with -s."""
import datetime
import os
import queue
import socket
import traceback

import numpy as np
import pytest
import torch

from learner_ref import CLIP, COEFF, Checks, decisive_pool, layer_scale, maxabs, params64, ref_forward, ref_losses

pytestmark = pytest.mark.gpu

EPOCHS = 2
POOL = 800


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def schedule(counts, bs, drop_last):
    """rows of every rank in every step of an epoch (parallel.plan_minibatches' rule, restated): drop_last takes
    min_r(n_r // bs) full minibatches, otherwise max_r(ceil(n_r / bs)) with short or empty ones"""
    steps = min(c // bs for c in counts) if drop_last else max(-(-c // bs) for c in counts)
    return [[min(bs, max(0, c - i * bs)) for c in counts] for i in range(steps)]


def make_cases(G, pool):
    """stage 1 and stage 2 cases of G ranks, each without and with the overlapped all-reduce"""
    rs = np.random.RandomState(40 + G)
    cases = []
    for stage, rows, drops, bs in ((1, (300, 170, 50)[:G], (0, 0, 0)[:G], 128),
                                   (2, (300, 260, 230)[:G], (20, 7, 33)[:G], 64)):
        offs = np.concatenate([[0], np.cumsum(rows)])
        assert offs[-1] <= len(pool['adv'])
        # raw advantages of a different mean and spread per rank: a rank-local normalisation would differ
        adv = np.concatenate([pool['adv'][offs[r]:offs[r + 1]] * (1 + 0.5 * r) + 0.3 * r for r in range(G)])
        filt = [sorted(rs.choice(rows[r], drops[r], replace=False).tolist()) for r in range(G)]
        kept = [rows[r] - drops[r] for r in range(G)]
        perms = [[rs.permutation(kept[r]) for _ in range(EPOCHS)] for r in range(G)]
        for overlap in (0, 1):
            cases.append(dict(name=f'G={G} stage{stage} overlap={overlap}', stage=stage, rows=list(rows),
                              offs=offs.tolist(), filt=filt, perms=perms, bs=bs, overlap=overlap, adv=adv.astype(np.float32),
                              sizes=schedule(kept, bs, stage == 2)))
    return cases


def _same_on_every_rank(t):
    import torch.distributed as dist
    x = t.detach().contiguous().cpu().view(torch.int32)
    got = [torch.empty_like(x) for _ in range(dist.get_world_size())]
    dist.all_gather(got, x)
    return all(torch.equal(x, y) for y in got)


def _recording_adam():
    from rl_collision_avoidance_b200.model.net import Adam

    class RecordingAdam(Adam):
        """Adam that keeps policy.grad x grad_scale, the gradient every step applies"""

        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.record = []

        def step(self, grad_scale=1.0):
            self.record.append(self.policy.grad.double() * grad_scale)
            super().step(grad_scale)

    return RecordingAdam


def _policy(bs):
    from golden_inputs import synthetic_state_dict
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=bs)
    pol.load_state_dict({k: torch.as_tensor(v) for k, v in synthetic_state_dict().items()})
    return pol


def _update(pol, opt, case, rank, memory):
    from rl_collision_avoidance_b200.model.ppo import ppo_update_stage1, ppo_update_stage2
    kw = dict(batch_size=case['bs'], memory=memory, epoch=EPOCHS, coeff_entropy=COEFF, clip_value=CLIP,
              num_step=case['rows'][rank], num_env=1, frames=3, obs_size=512, act_size=2, process_group=True,
              permutations=case['perms'][rank])
    if case['stage'] == 1:
        ppo_update_stage1(pol, opt, **kw)
    else:
        ppo_update_stage2(pol, opt, filter_index=case['filt'][rank], **kw)


def _union_rows(case, e, i):
    """pool rows of every rank in step i of epoch e"""
    bs, out = case['bs'], []
    for r in range(len(case['rows'])):
        drop = set(case['filt'][r])
        kept = np.array([j for j in range(case['rows'][r]) if j not in drop])
        perm = kept[case['perms'][r][e]]
        out.append(perm[i * bs:i * bs + case['sizes'][i][r]] + case['offs'][r])
    return np.concatenate(out)


def _reference_checks(case, pool, record):
    """(what, error, bound) of every step's recorded gradient against float64 autograd over the union of the rows"""
    from golden_inputs import synthetic_state_dict
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.model.net import TENSORS
    lib = _lib.load()
    offsets = [int(lib.rlca_policy_param_offset(i)) for i in range(len(TENSORS) + 1)]
    adv64 = case['adv'].astype(np.float64)
    adv64 = (adv64 - adv64.mean()) / adv64.std()
    out = []
    steps = len(case['sizes'])
    for k, got in enumerate(record):
        e, i = divmod(k, steps)
        rows = _union_rows(case, e, i)
        d64 = lambda a: torch.from_numpy(np.ascontiguousarray(a[rows])).cuda().double()
        P = params64(synthetic_state_dict(), grad=True)
        v, mean, _ = ref_forward(P, d64(pool['obs']).view(-1, 3, 512), d64(pool['gs']))
        _, loss = ref_losses(P, v, mean, d64(pool['act']), d64(pool['old_lp']), d64(adv64), d64(pool['tgt']))
        loss.backward()
        grads = {name: P[name].grad for name, _ in TENSORS}
        worst = (-1.0, None, 0.0, 0.0)
        for j, (name, shape) in enumerate(TENSORS):
            view = got[offsets[j]:offsets[j] + P[name].numel()].view(shape)
            err, bound = maxabs(view - grads[name]), 5e-5 * layer_scale(grads, name)
            r = err / bound if bound > 0 else (0.0 if err == 0 else np.inf)
            if r > worst[0]:
                worst = (r, name, err, bound)
        out.append((f'{case["name"]} epoch {e} step {i} ({len(rows)} rows) gradient vs float64 (worst: {worst[1]})',
                     worst[2], worst[3]))
    return out


def _worker(rank, world, port, out, pool, cases):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(seconds=180))
    try:
        from rl_collision_avoidance_b200.model.net import Adam
        from rl_collision_avoidance_b200.model.ppo import normalize_advantages
        RecordingAdam = _recording_adam()
        res = []
        for case in cases:
            os.environ['RLCA_DP_OVERLAP'] = str(case['overlap'])
            lo, hi = case['offs'][rank], case['offs'][rank + 1]
            cu = lambda a: torch.from_numpy(np.ascontiguousarray(a[lo:hi])).cuda()
            gs = cu(pool['gs'])
            adv = torch.from_numpy(case['adv'][lo:hi]).cuda()
            n = hi - lo
            memory = (cu(pool['obs']), gs[:, :2].contiguous(), gs[:, 2:].contiguous(), cu(pool['act']), cu(pool['old_lp']),
                      cu(pool['tgt']), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda'), adv)
            # the advantages every rank normalises with the moments of all ranks' rollouts
            a64 = case['adv'].astype(np.float64)
            ref = torch.from_numpy(((a64 - a64.mean()) / a64.std())[lo:hi]).cuda()
            norm_err = maxabs(normalize_advantages(adv, True).double() - ref)
            # lr = 0: the gradients of every step, at the same parameters
            pol = _policy(case['bs'])
            opt = RecordingAdam(pol.parameters(), lr=0.0)
            _update(pol, opt, case, rank, memory)
            torch.cuda.synchronize()
            grads_same = all(_same_on_every_rank(g) for g in opt.record)
            checks = _reference_checks(case, pool, opt.record) if rank == 0 else []
            nsteps = len(opt.record)
            del opt, pol
            # a real learning rate: the replicas stay bit-identical
            pol = _policy(case['bs'])
            opt = Adam(pol.parameters(), lr=5e-5)
            _update(pol, opt, case, rank, memory)
            torch.cuda.synchronize()
            replicated = all(_same_on_every_rank(t) for t in (pol.flat, opt.exp_avg, opt.exp_avg_sq))
            moved = bool((pol.flat != _policy(case['bs']).flat).any())
            res.append(dict(name=case['name'], norm_err=norm_err, grads_same=grads_same, checks=checks, nsteps=nsteps,
                            adam_steps=opt.step_count, replicated=replicated, moved=moved))
            del opt, pol
        out.put((rank, res, None))
    except BaseException:
        out.put((rank, None, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('G', [2, 3])
def test_ppo_update_process_group_on_one_gpu(built, G):
    import torch.multiprocessing as mp
    pool = decisive_pool(POOL)
    pool = {k: pool[k] for k in ('obs', 'gs', 'act', 'old_lp', 'tgt', 'adv')}
    pool['obs'] = pool['obs'].reshape(POOL, 1536)
    cases = make_cases(G, pool)
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, G, port, q, pool, cases)) for r in range(G)]
    try:
        for p in procs:
            p.start()
        res = {}
        for _ in procs:
            try:
                rank, r, err = q.get(timeout=600)
            except queue.Empty:
                pytest.fail('a worker did not report within 600 s')
            assert err is None, f'rank {rank} failed:\n{err}'
            res[rank] = r
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0, f'a worker exited with {p.exitcode}'
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
            if p.is_alive():
                p.kill()
                p.join()
    check = Checks()
    for ci, case in enumerate(cases):
        expect = EPOCHS * len(case['sizes'])
        for rank in range(G):
            got = res[rank][ci]
            assert got['name'] == case['name']
            check(f'{case["name"]} rank {rank} advantage normalisation vs float64', got['norm_err'], 1e-6)
            if got['nsteps'] != expect or got['adam_steps'] != expect:
                check.failed.append(f'{case["name"]} rank {rank}: {got["nsteps"]} / {got["adam_steps"]} optimizer steps, '
                                    f'the schedule has {expect}')
            if not got['grads_same']:
                check.failed.append(f'{case["name"]} rank {rank}: the gradient Adam applies differs between ranks')
            if not got['replicated']:
                check.failed.append(f'{case["name"]} rank {rank}: parameters or moments differ between ranks after '
                                    f'training at lr 5e-5')
            if not got['moved']:
                check.failed.append(f'{case["name"]} rank {rank}: training at lr 5e-5 left the parameters unchanged')
        for what, err, bound in res[0][ci]['checks']:
            check(what, err, bound)
        assert len(res[0][ci]['checks']) == expect
    # the cases reach the branches they are for
    s1 = cases[0]['sizes']
    assert any(0 < sz < cases[0]['bs'] for step in s1 for sz in step) and any(0 in step for step in s1)
    check.done()
