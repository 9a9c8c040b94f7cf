"""Multi-GPU plumbing (SURVEY.md §8(e)): one process per GPU, worlds sharded contiguously, no data-path
collective for the env tick; the learner all-reduces (1) three advantage moments per update and (2) the flat
gradient buffer per optimizer step.  Everything here works on whatever device the tensors live on, so the
host-side logic is exercised by world_size-2 gloo tests on CPU (tests/test_parallel_gloo.py)."""
from __future__ import annotations

import torch


def shard_worlds(total_worlds: int, rank: int, world_size: int):
    """Contiguous split of `total_worlds` worlds: returns (world_offset, num_worlds) of this rank.
    The first (total % world_size) ranks take one extra world."""
    if not (0 <= rank < world_size):
        raise ValueError('rank out of range')
    base, rem = divmod(total_worlds, world_size)
    count = base + (1 if rank < rem else 0)
    offset = rank * base + min(rank, rem)
    return offset, count


def allreduce_moments(moments: torch.Tensor, group=None):
    """moments = (sum, sum of squares, count) in float64; summed over ranks in place."""
    import torch.distributed as dist
    dist.all_reduce(moments, op=dist.ReduceOp.SUM, group=group)
    return moments


def allreduce_diagnostics(acc: torch.Tensor, rules, group=None):
    """Accumulator rows (..., columns) merged over ranks in place, column c by rules[c]: 'sum' columns with SUM, 'max'
    columns with MAX and 'min' columns, negated, with the same MAX (model/diagnostics.py).  Every rank ends with the
    same rows, so a decision taken from them is the same everywhere."""
    import torch.distributed as dist
    idx = lambda rule: torch.tensor([c for c, r in enumerate(rules) if r == rule], dtype=torch.long, device=acc.device)
    isum, imax, imin = idx('sum'), idx('max'), idx('min')
    sums = acc[..., isum].contiguous()
    dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=group)
    ext = torch.cat((acc[..., imax], -acc[..., imin]), dim=-1).contiguous()
    dist.all_reduce(ext, op=dist.ReduceOp.MAX, group=group)
    acc[..., isum] = sums
    acc[..., imax] = ext[..., :imax.numel()]
    acc[..., imin] = -ext[..., imax.numel():]
    return acc


def normalize_from_moments(x: torch.Tensor, moments: torch.Tensor):
    """(x - mean) / std with numpy semantics (ddof = 0) from global moments (model/ppo.py:148)."""
    cnt = moments[2]
    mean = moments[0] / cnt
    var = moments[1] / cnt - mean * mean
    return ((x.double() - mean) / torch.sqrt(var)).to(x.dtype)


def average_gradients(flat_grad: torch.Tensor, group=None):
    """Sum the flat gradient over ranks (the 1/world_size is folded into the fused Adam step)."""
    import torch.distributed as dist
    dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    return flat_grad


def broadcast_parameters(flat: torch.Tensor, src=0, group=None):
    import torch.distributed as dist
    dist.broadcast(flat, src=src, group=group)
    return flat


def plan_minibatches(n_local: int, batch_size: int, drop_last: bool, group=None, distributed: bool = False):
    """Agree on ONE minibatch schedule per epoch across ranks whose row counts differ (stage 2 deletes the rows of
    `filter_index` per rank, model/ppo.py:212-218; uneven world shards give different T*N per rank).

    Every rank must issue the same number of gradient all-reduces, so the step count is global:
      drop_last (stage 2, model/ppo.py:221-223): steps = min over ranks of n_r // batch_size; every minibatch is full,
          a rank with more rows drops a longer (random, re-drawn every epoch) tail - the reference's own rule applied
          to the rank that binds;
      otherwise (stage 1, :159-160): steps = max over ranks of ceil(n_r / batch_size); a rank that runs out of rows
          takes a short or EMPTY minibatch (zero gradient, still all-reduces).
    Returns (steps, sizes, weights): sizes[i] = rows this rank uses in step i, weights[i] = sizes[i] * world /
    sum over ranks of sizes[i], the factor that makes (all-reduced gradient / world) the mean over all rows of the
    global minibatch (rlca_ppo_loss_fwd_bwd_weighted)."""
    counts = [int(n_local)]
    rank = 0
    if distributed:
        import torch.distributed as dist
        world = dist.get_world_size(group)
        rank = dist.get_rank(group)
        t = torch.zeros(world, dtype=torch.int64)
        t[rank] = int(n_local)
        backend = dist.get_backend(group)
        if backend == 'nccl':
            t = t.cuda()
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        counts = [int(x) for x in t.cpu().tolist()]
    world = len(counts)
    bs = int(batch_size)
    if drop_last:
        steps = min(c // bs for c in counts)
    else:
        steps = max((c + bs - 1) // bs for c in counts)
    sizes, weights = [], []
    for i in range(steps):
        per_rank = [min(bs, max(0, c - i * bs)) for c in counts]
        tot = sum(per_rank)
        sizes.append(per_rank[rank])
        weights.append(per_rank[rank] * world / tot if tot else 0.0)
    return steps, sizes, weights


def agree_to_stop(local_stop: bool, device=None, group=None) -> bool:
    """True on every rank as soon as ANY rank wants to leave the training loop (the exit test uses rank-local episode
    counts; a rank that left alone would strand the others in the next all-reduce)."""
    import torch.distributed as dist
    t = torch.tensor([1.0 if local_stop else 0.0], device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return bool(t.item() > 0)


def grad_buckets(offsets):
    """(early, late) index ranges of the flat gradient buffer.  early = everything outside the conv towers (tensors
    5..12 and 17..22 of the state_dict order: fc1, fc2, heads - 97 % of the floats), final before the conv tower
    backward starts; late = logstd + the four conv tensors of each tower."""
    early = [(offsets[5], offsets[13]), (offsets[17], offsets[23])]
    late = [(offsets[0], offsets[5]), (offsets[13], offsets[17])]
    return early, late


class OverlappedGradSync:
    """All-reduce of the flat gradient that hides most of the transfer under the backward pass: librlca records an
    event when the fc-side gradients are final (rlca_policy_set_grad_event); their ranges are all-reduced from a side
    stream while the dF GEMM and the conv tower backward still run, the small conv ranges afterwards.  Results are
    those of one all-reduce of the whole buffer (sum; the 1/world_size goes into the fused Adam step)."""

    def __init__(self, policy, group=None):
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        self.policy = policy
        self.early, self.late = grad_buckets(policy.offsets)
        self.cuda = policy.grad.is_cuda
        if self.cuda:
            from . import _lib
            import ctypes as C
            self.side = torch.cuda.Stream(device=policy.device)
            self.event = torch.cuda.Event(enable_timing=False)
            self.event.record(torch.cuda.current_stream(policy.device))       # creates the underlying cudaEvent_t
            self._handle = C.c_void_p(self.event.cuda_event)
            self._lib = _lib
            self.attach()

    def attach(self):
        """(Re-)register the event with the policy's current workspace (a workspace is rebuilt when max_batch grows)."""
        if self.cuda:
            self._ws = self.policy._workspace(1)
            self._lib.check(self.policy.lib.rlca_policy_set_grad_event(self._ws, self._handle))

    def reduce(self):
        """Call right after rlca_policy_backward on the current stream; returns when the current stream is ordered after
        every all-reduce."""
        g = self.policy.grad
        if not self.cuda:
            for a, b in self.early + self.late:
                self.dist.all_reduce(g[a:b], group=self.group)
            return
        if self.policy._ws is not self._ws:
            self.attach()
        main = torch.cuda.current_stream(g.device)
        self.side.wait_event(self.event)
        with torch.cuda.stream(self.side):
            works = [self.dist.all_reduce(g[a:b], group=self.group, async_op=True) for a, b in self.early]
        for a, b in self.late:
            self.dist.all_reduce(g[a:b], group=self.group)
        for w in works:
            w.wait()
        main.wait_stream(self.side)

    def mark_ready(self):
        """The whole buffer is final on the current stream without a backward pass (e.g. zeroed for an empty minibatch)."""
        if self.cuda:
            self.event.record(torch.cuda.current_stream(self.policy.grad.device))

    def close(self):
        if self.cuda:
            self._lib.check(self.policy.lib.rlca_policy_set_grad_event(self.policy._workspace(1), None))


class PeerAdam:
    """Data-parallel optimizer step as ONE kernel over NVLink peer memory (csrc/rlca_dp.cu): reduce-scatter of the flat
    gradient + Adam + all-gather of the parameter and both moments, instead of an NCCL all-reduce followed by the Adam
    kernel (the reference takes an optimizer step per minibatch, model/ppo.py:186-188, so the collective is on the
    critical path of every step).  The four flat buffers of the policy / optimizer move into one symmetric-memory
    allocation (torch.distributed._symmetric_memory: peer mappings of every rank's buffer, the NVSwitch multicast
    mapping when the fabric offers one, and cross-GPU barriers); rank r updates shard r and writes the new parameters
    into every rank's buffer, so the weights stay replicated bit for bit.  The Adam moments are sharded (rank r owns
    those of shard r; `gather_moments()` reads them back through the peer mappings for a checkpoint) unless
    `replicate_moments=True`.

        opt = Adam(policy.parameters(), lr)
        PeerAdam.attach(policy, opt)          # after init_process_group('nccl'); raises if peer memory is unavailable
        ... backward ...; opt.step(grad_scale=1 / world)     # no separate gradient all-reduce
    """

    def __init__(self, policy, optimizer, group=None, replicate_moments=False):
        import ctypes as C
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        self.replicate = bool(replicate_moments)
        from . import _lib
        self._lib, self._C = _lib, C
        group = group if group is not None else dist.group.WORLD
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        n = policy.flat_size
        if n % 4:
            raise ValueError('flat buffer size must be a multiple of 4 floats')
        self.n = n
        self.buf = symm_mem.empty(4 * n, dtype=torch.float32, device=policy.device)
        self.buf.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, group)
        grad, flat = self.buf[0:n], self.buf[n:2 * n]
        m, v = self.buf[2 * n:3 * n], self.buf[3 * n:4 * n]
        m.copy_(optimizer.exp_avg)
        v.copy_(optimizer.exp_avg_sq)
        policy.rebind_storage(flat, grad)
        optimizer.exp_avg, optimizer.exp_avg_sq = m, v
        base = [int(x) for x in self.hdl.buffer_ptrs]
        arr = C.c_uint64 * self.world
        self._grad = arr(*[b for b in base])
        self._param = arr(*[b + 4 * n for b in base])
        self._m = arr(*[b + 8 * n for b in base])
        self._v = arr(*[b + 12 * n for b in base])
        mc = int(getattr(self.hdl, 'multicast_ptr', 0) or 0)
        self.nvls = mc != 0
        self._mc = [mc + k * 4 * n if mc else 0 for k in range(4)]
        self.policy = policy
        torch.cuda.synchronize(policy.device)
        self.hdl.barrier(channel=0)                      # everybody's buffers are in place before anybody steps

    @classmethod
    def attach(cls, policy, optimizer, group=None, replicate_moments=False):
        optimizer.peer = cls(policy, optimizer, group, replicate_moments)
        return optimizer.peer

    def shard(self, r):
        chunk = ((self.n // 4 + self.world - 1) // self.world) * 4
        lo = min(r * chunk, self.n)
        return lo, min(lo + chunk, self.n)

    def gather_moments(self):
        """(exp_avg, exp_avg_sq) of the whole buffer on this rank: every shard read from its owner through the peer
        mapping (no collective: call it when no optimizer step is in flight, e.g. between updates)."""
        torch.cuda.synchronize(self.policy.device)
        n = self.n
        m, v = self.buf[2 * n:3 * n].clone(), self.buf[3 * n:4 * n].clone()
        if not self.replicate:
            for r in range(self.world):
                if r == self.rank:
                    continue
                lo, hi = self.shard(r)
                remote = self.hdl.get_buffer(r, (4 * n,), torch.float32)
                m[lo:hi].copy_(remote[2 * n + lo:2 * n + hi])
                v[lo:hi].copy_(remote[3 * n + lo:3 * n + hi])
        return m, v

    def step(self, opt, grad_scale):
        p = self.policy
        self.hdl.barrier(channel=0)                      # every rank's gradient is complete
        self._lib.check(p.lib.rlca_adam_step_allreduce(
            self._grad, self._param, self._m, self._v, self._mc[0], self._mc[1], self._mc[2], self._mc[3],
            self.rank, self.world, self.n, opt.lr, opt.betas[0], opt.betas[1], opt.eps, opt.step_count, grad_scale,
            int(self.replicate), p._stream()))
        self.hdl.barrier(channel=1)                      # every shard has landed everywhere
