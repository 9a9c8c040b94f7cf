"""Fused data-parallel optimizer step over NVLink peer memory (csrc/rlca_dp.cu, parallel.PeerAdam) against the
two-call path it replaces: NCCL all-reduce of the flat gradient + rlca_adam_step with grad_scale = 1 / world.
Needs 2 GPUs (python -m pytest tests/test_dp_peer_gpu.py -m gpu on a 2-GPU machine); skipped on one."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    try:
        from rl_collision_avoidance_b200 import _lib
        from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy, _ptr
        from rl_collision_avoidance_b200.parallel import PeerAdam
        pol = CNNPolicy(device=str(dev), seed=3, max_batch=8)
        opt = Adam(pol.parameters(), lr=5e-5)
        peer = PeerAdam.attach(pol, opt)
        gen = torch.Generator(device=dev)
        gen.manual_seed(100 + rank)
        # reference copies
        p_ref, m_ref, v_ref = pol.flat.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone()
        ok_vals, ok_rep = True, True
        for step in range(1, 4):
            pol.grad.copy_(torch.randn(pol.flat_size, device=dev, generator=gen) * (0.1 * step))
            g_ref = pol.grad.clone()
            dist.all_reduce(g_ref)
            _lib.check(pol.lib.rlca_adam_step(_ptr(p_ref), _ptr(g_ref), _ptr(m_ref), _ptr(v_ref), pol.flat_size, opt.lr,
                                              opt.betas[0], opt.betas[1], opt.eps, step, 1.0 / world, pol._stream()))
            opt.step(grad_scale=1.0 / world)
            torch.cuda.synchronize(dev)
            # world = 2: a + b is the same float whichever rank (or the switch) adds it -> bit-exact
            gm, gv = opt.state_dict()['exp_avg'], opt.state_dict()['exp_avg_sq']      # sharded moments, gathered over P2P
            same = torch.equal(pol.flat, p_ref) and torch.equal(gm, m_ref) and torch.equal(gv, v_ref)
            close = (pol.flat - p_ref).abs().max().item() < 1e-6 and (gm - m_ref).abs().max().item() < 1e-6
            dist.barrier()                        # nobody steps again while a peer is still reading its shard
            ok_vals = ok_vals and (same if world == 2 else close)
            # replicated state: every rank holds the same bits
            chk = torch.stack([pol.flat.double().sum(), gm.double().sum(), gv.double().sum()])
            lo, hi = chk.clone(), chk.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN)
            dist.all_reduce(hi, op=dist.ReduceOp.MAX)
            ok_rep = ok_rep and bool(torch.equal(lo, hi))
        # the named views follow the moved storage, checkpoints see the updated weights
        sd = pol.state_dict()
        ok_views = torch.equal(sd['act_fc1.weight'].reshape(-1), pol.flat[pol.offsets[5]:pol.offsets[5] + 256 * 4096])
        out.put((rank, ok_vals, ok_rep, ok_views, peer.nvls, opt.step_count))
    finally:
        dist.destroy_process_group()


def test_peer_adam_matches_allreduce_plus_adam(built):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ok_vals, ok_rep, ok_views, nvls, steps in res:
        assert ok_vals, f'rank {rank}: fused step differs from all-reduce + Adam'
        assert ok_rep, f'rank {rank}: state not replicated across ranks'
        assert ok_views and steps == 3
    print('NVLS multicast:', res[0][4])
