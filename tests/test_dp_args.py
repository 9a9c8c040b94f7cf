"""Host side of the data-parallel optimizer step (csrc/rlca_dp.cu): the arguments rlca_adam_step_allreduce rejects
before it touches the device, and the shard rule that PeerAdam shares with the kernel.  No GPU needed."""
import ctypes as C

import pytest
import torch

from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.parallel import PeerAdam

RLCA_ERR_INVALID = 1


def kernel_shard(n, world, rank):
    """the kernel's rule: chunk = ceil(n / 4 / world) * 4 floats, rank r owns [r * chunk, (r + 1) * chunk) clipped to n"""
    chunk = -(-(n // 4) // world) * 4
    lo = min(rank * chunk, n)
    return lo, min(lo + chunk, n)


def peer_shard(n, world, rank):
    pa = PeerAdam.__new__(PeerAdam)           # only the fields shard() reads: no process group, no symmetric memory
    pa.n, pa.world = n, world
    return pa.shard(rank)


@pytest.mark.parametrize('world', range(1, 17))
def test_shards_partition_the_buffer(world):
    """PeerAdam.shard gives every float of [0, n) to exactly one rank, in rank order, each shard a multiple of 4 long
    (trailing ranks may get an empty shard), and agrees with the kernel's rule."""
    for n in (4, 8, 12, 16, 60, 64, 1028, 4 * world, 4 * world + 4, 4 * world - 4, 2172160, 2172160 + 4 * world - 4):
        if n < 4:
            continue
        spans = [peer_shard(n, world, r) for r in range(world)]
        assert spans == [kernel_shard(n, world, r) for r in range(world)], (n, world)
        assert spans[0][0] == 0 and spans[-1][1] == n, (n, world)
        for (lo, hi), (lo2, _) in zip(spans[:-1], spans[1:]):
            assert hi == lo2, (n, world, spans)
        assert all(lo <= hi and lo % 4 == 0 and hi % 4 == 0 for lo, hi in spans), (n, world, spans)
        # no rank gets more than ceil(n / 4 / world) float4s, so the largest shard bounds the step's latency
        assert max(hi - lo for lo, hi in spans) == kernel_shard(n, world, 0)[1], (n, world)
    # the cases the GPU tests rely on
    assert [peer_shard(8, 16, r) for r in range(16)] == [(0, 4), (4, 8)] + [(8, 8)] * 14
    assert [peer_shard(12, 2, r) for r in range(2)] == [(0, 8), (8, 12)]


def test_adam_step_allreduce_rejects_bad_arguments(built):
    """Each rejected call returns RLCA_ERR_INVALID before anything is launched: on a machine without a GPU an accepted
    call would fail at the launch with a CUDA error instead."""
    lib = _lib.load()
    world, n = 2, 64
    have_gpu = torch.cuda.is_available()
    if have_gpu:   # real buffers, so that the accepted control call below runs a harmless step on zeros
        bufs = [torch.zeros(n, device='cuda') for _ in range(4 * world)]
        addrs = [b.data_ptr() for b in bufs]
    else:          # never dereferenced: every call but the control returns before the launch
        addrs = [0x10000 * (k + 1) for k in range(4 * world)]
    arr = lambda xs: (C.c_uint64 * len(xs))(*xs)
    good = [arr(addrs[k * world:(k + 1) * world]) for k in range(4)]

    def call(ptrs=None, rank=0, world_=world, n_=n, step=1):
        p = good if ptrs is None else ptrs
        return lib.rlca_adam_step_allreduce(*p, 0, 0, 0, 0, rank, world_, n_, 1e-3, 0.9, 0.999, 1e-8, step,
                                            1.0 / world, 0, None)

    bad = {'world 0': dict(world_=0), 'world 17': dict(world_=17), 'world -1': dict(world_=-1),
           'rank = world': dict(rank=world), 'rank > world': dict(rank=world + 3), 'rank -1': dict(rank=-1),
           'n % 4 = 2': dict(n_=62), 'n % 4 = 1': dict(n_=61), 'n 0': dict(n_=0), 'n -4': dict(n_=-4),
           'step 0': dict(step=0), 'step -1': dict(step=-1)}
    for k in range(4):
        bad[f'NULL array {k}'] = dict(ptrs=[None if j == k else good[j] for j in range(4)])
        for q in range(world):
            entries = list(addrs[k * world:(k + 1) * world])
            entries[q] = 0
            bad[f'NULL entry {q} of array {k}'] = dict(ptrs=[arr(entries) if j == k else good[j] for j in range(4)])
    for what, kw in bad.items():
        assert call(**kw) == RLCA_ERR_INVALID, what
        msg = lib.rlca_last_error()
        assert msg and (b'rlca_adam_step_allreduce' in msg or b'NULL' in msg), (what, msg)
    if have_gpu:
        assert call() == 0
        torch.cuda.synchronize()
        assert all(bool((b == 0).all()) for b in bufs)
    else:
        assert call() not in (0, RLCA_ERR_INVALID), 'a valid call on a machine without a GPU must fail at the launch'
