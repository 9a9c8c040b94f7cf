"""The paper's SL-policy baseline (DESIGN.md §9g): the CNNPolicy network trained by supervised learning on an expert's
demonstrations, the expert being one of the baseline controllers of orca.py.

    obs, gs, action = collect(env, NhOrcaController(env, obstacles=True), samples=100000)
    rows = sl_update(policy, Adam(policy.parameters(), lr), (obs, gs, action), batch_size=1024, epochs=1)
    held_out = sl_loss(policy, (obs, gs, action), batch_size=1024, rows=index)

Recording (rlca_demo_append), the minibatch gather, the forward, the behaviour-cloning loss (rlca_bc_loss_fwd_bwd),
the backward and Adam all run in librlca.so; the loops below only order them and synchronise once per call.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .model.net import CNNPolicy, _ptr
from .model.ppo import _MinibatchGather, _stream

LASER_HIST = 3


class DemoSet:
    """A fixed-capacity dataset of (scan stack, goal | speed, clipped action) rows on the env's device, appended to by
    rlca_demo_append without host synchronisation.  `count()` synchronises."""

    def __init__(self, env, capacity):
        if int(capacity) < 1:
            raise ValueError('capacity must be >= 1')
        self.env, self.capacity = env, int(capacity)
        dev = env.device
        self.obs = torch.empty(self.capacity, LASER_HIST * env.beam_mum, device=dev)
        self.gs = torch.empty(self.capacity, 4, device=dev)
        self.action = torch.empty(self.capacity, 2, device=dev)
        self.counter = torch.zeros(2, dtype=torch.int64, device=dev)       # rows held, completion ticket
        self._set = _lib.DemoSet(_ptr(self.obs), _ptr(self.gs), _ptr(self.action), _ptr(self.counter), self.capacity)

    def append(self, action, stack, prev_flags=None):
        """Record the tick `env.control_vel(action, stack_in=stack, ...)` is about to run: call it before that tick.
        `prev_flags` are the previous tick's flags (auto_reset 0 only; None = no agent was done)."""
        env = self.env
        io = _lib.StepIO(_ptr(action), None, None, None, _ptr(prev_flags), _ptr(env.gs), None, _ptr(stack), None)
        _lib.check(env.lib.rlca_demo_append(C.byref(env.cfg), C.byref(env._state_struct(env._cur)), C.byref(io),
                                            C.byref(self._set), env._stream()))

    def count(self):
        return int(self.counter[0])

    def rows(self):
        """(obs (n, 3 * beams), gs (n, 4), action (n, 2)) views of the rows held."""
        n = self.count()
        return self.obs[:n], self.gs[:n], self.action[:n]


def collect(env, controller, samples, record_every=1, check_every=50):
    """Drive every robot of `env` with `controller` (a callable returning the (N, 2) raw action, e.g. an
    NhOrcaController) from a fresh reset, as evaluation.evaluate does (auto_reset 0: v = 0 after termination), and
    record every `record_every`-th tick until `samples` rows are held.  A row is recorded for each agent whose action
    drives an episode that has not ended (rlca_demo_append).  On the circle (auto_reset 0), which runs one episode,
    recording stops early when every robot is done.  The count is checked every `check_every` ticks once enough ticks
    have run to fill the dataset.  Returns device tensors obs (n, 3 * beams), gs (n, 4), action (n, 2), n <= samples."""
    if int(record_every) < 1 or int(check_every) < 1:
        raise ValueError('record_every and check_every must be >= 1')
    demo = DemoSet(env, samples)
    N, dev = env.N, env.device
    circle = int(env.cfg.auto_reset) == 0
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    if env.sc.layout is not None:
        env.random_layout()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(N, 3, env.beam_mum, device=dev)]
    terminal = torch.zeros(N, dtype=torch.bool, device=dev)
    first_check = -(-demo.capacity // N) * int(record_every)      # ticks before the dataset can be full
    tick = 0
    while True:
        k = tick & 1
        action = controller()
        if tick % record_every == 0:
            demo.append(action, stacks[k], env.flags if circle and tick > 0 else None)
        scaled = action
        if circle:
            scaled = torch.stack((torch.where(terminal, 0.0, action[:, 0]), action[:, 1]), 1)
        env.control_vel(scaled, stack_in=stacks[k], stack_out=stacks[1 - k])
        if circle:
            terminal = env.flags[:, 0] != 0
        tick += 1
        if tick % check_every == 0 and (circle or tick >= first_check):
            if demo.count() >= demo.capacity or (circle and bool(terminal.all())):
                break
    return demo.rows()


def _minibatches(n, bs):
    return [min(bs, n - b0) for b0 in range(0, n, bs)]


def sl_update(policy: CNNPolicy, optimizer, data, batch_size, epochs, generator=None, rows=None):
    """`epochs` passes of behaviour cloning over `data` = (obs (n, 3 * beams), gs (n, 4), action (n, 2)), or over its
    rows `rows` (an index tensor): per epoch a random permutation (torch.randperm with `generator`), minibatches of
    `batch_size` rows in its order (the last one ragged), each gathered in one launch (rlca_gather_minibatch), then
    forward, BC loss, backward and one fused Adam step.  Returns the per-minibatch losses, logged on the device and
    read once at the end."""
    lib = _lib.load()
    obs, gs, act = (t.float().contiguous() for t in data)
    dev = policy.device
    keep = torch.arange(obs.shape[0], device=dev) if rows is None else rows.to(device=dev, dtype=torch.long)
    n, bs = keep.numel(), int(batch_size)
    if n < 1 or bs < 1 or int(epochs) < 1:
        raise ValueError('sl_update needs rows, batch_size >= 1 and epochs >= 1')
    sizes = _minibatches(n, bs)
    b_obs = torch.empty(bs, obs.shape[1], device=dev)
    b_gs = torch.empty(bs, 4, device=dev)
    b_act = torch.empty(bs, 2, device=dev)
    v = torch.empty(bs, device=dev)
    mean = torch.empty(bs, 2, device=dev)
    log = torch.zeros(int(epochs) * len(sizes), device=dev)
    ws = policy._workspace(bs)
    st = _stream(dev)
    gather = _MinibatchGather(lib, (obs, gs, act), (b_obs, b_gs, b_act), (obs.shape[1], 4, 2), dev)
    k = 0
    for _ in range(int(epochs)):
        perm = keep[torch.randperm(n, device=dev, generator=generator)]
        for bi, nb in enumerate(sizes):
            gather(perm[bi * bs:bi * bs + nb].contiguous())
            _lib.check(lib.rlca_policy_forward(ws, _ptr(policy.flat), _ptr(b_obs), _ptr(b_gs), nb, _ptr(v), _ptr(mean), st))
            _lib.check(lib.rlca_bc_loss_fwd_bwd(ws, _ptr(policy.flat), _ptr(mean), _ptr(b_act), nb, _ptr(log[k:k + 1]), st))
            _lib.check(lib.rlca_policy_backward(ws, _ptr(policy.flat), _ptr(b_obs), _ptr(b_gs), nb, _ptr(policy.grad), st))
            optimizer.step()
            k += 1
    return log.cpu().tolist()


def sl_loss(policy: CNNPolicy, data, batch_size, rows=None):
    """The BC loss of the whole of `data` (or of its rows `rows`) under the current parameters, without a gradient
    step: the row-weighted mean of the minibatch losses, in `rows` order."""
    lib = _lib.load()
    obs, gs, act = (t.float().contiguous() for t in data)
    dev = policy.device
    keep = torch.arange(obs.shape[0], device=dev) if rows is None else rows.to(device=dev, dtype=torch.long)
    n, bs = keep.numel(), int(batch_size)
    if n < 1 or bs < 1:
        raise ValueError('sl_loss needs rows and batch_size >= 1')
    sizes = _minibatches(n, bs)
    b_obs = torch.empty(bs, obs.shape[1], device=dev)
    b_gs = torch.empty(bs, 4, device=dev)
    b_act = torch.empty(bs, 2, device=dev)
    v = torch.empty(bs, device=dev)
    mean = torch.empty(bs, 2, device=dev)
    log = torch.zeros(len(sizes), device=dev)
    ws = policy._workspace(bs)
    st = _stream(dev)
    gather = _MinibatchGather(lib, (obs, gs, act), (b_obs, b_gs, b_act), (obs.shape[1], 4, 2), dev)
    for bi, nb in enumerate(sizes):
        gather(keep[bi * bs:bi * bs + nb].contiguous())
        _lib.check(lib.rlca_policy_forward(ws, _ptr(policy.flat), _ptr(b_obs), _ptr(b_gs), nb, _ptr(v), _ptr(mean), st))
        _lib.check(lib.rlca_bc_loss_fwd_bwd(ws, _ptr(policy.flat), _ptr(mean), _ptr(b_act), nb, _ptr(log[bi:bi + 1]), st))
    w = torch.tensor(sizes, dtype=torch.float64, device=dev)
    return float((log.double() * w).sum() / n)
