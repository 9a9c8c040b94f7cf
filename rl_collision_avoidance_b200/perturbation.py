"""The perturbations between a controller and the robots (DESIGN.md §9y): `Chain`, the one order in which evaluate()
and the trainer apply noise (§9p), latency (§9q), acceleration limits (§9r), localization error (§9s) and the global
planner (§9w, §9x), and the plumbing the four perturbation modules share.

    chain = Chain(env, noise, latency, dynamics, localization, planner)     # any link may be None
    gs = chain.sense(stacks[0])                     # the start: every row starts an episode
    executed = chain.command(scaled, None)          # the first tick: no flags of a previous tick
    env.control_vel(executed, stack_in=stacks[0], stack_out=stacks[1])
    gs = chain.sense(stacks[1], env.flags)          # after the tick
    executed = chain.command(scaled, env.flags)     # every later tick: the flags of the tick before
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

MAX_STREAM_ID = (1 << 24) - 1


class Chain:
    """The perturbations of one env handle; each link is optional.  On the command side latency delays the command,
    noise perturbs the delayed one and the acceleration limits act last, so that their state is what the tick executes;
    latency and the limits take the flags of the previous tick.  On the sensing side latency replaces the newest frame
    with the true frame of d ticks earlier, noise perturbs what is delivered, localization turns the true gs into the
    believed one and the planner replaces the local goal last; all four take the flags of the tick just run (None at
    the start).  Each link is called exactly as its own interface documents, so its draw counters advance as they would
    if the caller called it directly."""

    def __init__(self, env, noise=None, latency=None, dynamics=None, localization=None, planner=None):
        for name, link in (('noise', noise), ('latency', latency), ('dynamics', dynamics),
                           ('localization', localization), ('planner', planner)):
            if link is not None and link.env is not env:
                raise ValueError(f'the {name} belongs to another env')
        if planner is not None and planner.steer and localization is not None:
            raise ValueError('the planner plans from the true pose; localization error needs a planner on the '
                             'believed pose')
        self.env = env
        self.noise, self.latency, self.dynamics = noise, latency, dynamics
        self.localization, self.planner = localization, planner

    def command(self, cmd, prev_flags):
        """Before a tick: the command the robots execute for the issued command `cmd` (not written).  `prev_flags` are
        those of the previous tick, None on a run's first tick."""
        if self.latency is not None:
            cmd = self.latency.action(cmd, prev_flags)
        if self.noise is not None:
            cmd = self.noise.action(cmd)
        if self.dynamics is not None:
            cmd = self.dynamics.action(cmd, prev_flags)
        return cmd

    def sense(self, stack, flags=None, gs=None, reward=None, eplog=None):
        """After a tick and any re-layout, with its flags (None at a run's start): perturb the newest frame of `stack`
        in place and return the gs the policy reads.  With `gs` (the slot the tick wrote) localization and the planner
        write into it in place, and a reward planner shapes `reward` and `eplog` in place.  Without, they read env.gs
        and return buffers of their own; None when the policy reads env.gs."""
        if self.latency is not None:
            self.latency.scan(stack, flags)
        if self.noise is not None:
            self.noise.scan(stack, flags)
        out = gs
        if self.localization is not None:
            out = self.localization.observe(flags, gs=gs, out=gs)
        if self.planner is not None:
            planned = self.planner.update(flags, reward, eplog, gs=gs)
            if self.planner.steer:
                out = planned
        return out

    def settings(self):
        """{name: settings} of the links noise, latency, dynamics and localization that are present"""
        links = (('noise', self.noise), ('latency', self.latency), ('dynamics', self.dynamics),
                 ('localization', self.localization))
        return {name: link.settings() for name, link in links if link is not None}


# ------------------------------------------------------------------------------------------------ shared plumbing
def check_stream_id(stream_id):
    if isinstance(stream_id, bool) or int(stream_id) != stream_id or not 0 <= int(stream_id) <= MAX_STREAM_ID:
        raise ValueError(f'stream_id must be an integer in 0 .. {MAX_STREAM_ID}, got {stream_id!r}')
    return int(stream_id)


def check_seed(kind, seed):
    """`seed` as an int; ValueError naming the `kind` of seed unless it is an integer in 0 .. 2^64 - 1"""
    if isinstance(seed, bool) or int(seed) != seed or not 0 <= int(seed) < 1 << 64:
        raise ValueError(f'the {kind} seed must be an integer in 0 .. 2^64 - 1, got {seed!r}')
    return int(seed)


def device_of(env):
    """The torch.device of `env`, with the current CUDA device's index when env.device names none"""
    d = torch.device(env.device)
    return d if d.index is not None or d.type != 'cuda' else torch.device('cuda', torch.cuda.current_device())


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def check_stack(env, dev, stack):
    """ValueError unless `stack` is a contiguous (env.N, 3, beams) float32 tensor on the device `dev` of `env`"""
    if tuple(stack.shape) != (env.N, 3, env.beam_mum) or stack.dtype != torch.float32 or \
            not stack.is_contiguous() or stack.device != dev:
        raise ValueError(f'stack must be a contiguous ({env.N}, 3, {env.beam_mum}) float32 tensor on {env.device}')


def check_flags(env, dev, flags):
    """ValueError unless `flags` is None or a contiguous (env.N, 4) uint8 tensor on the device `dev` of `env`"""
    if flags is not None and (tuple(flags.shape) != (env.N, 4) or flags.dtype != torch.uint8 or
                              not flags.is_contiguous() or flags.device != dev):
        raise ValueError(f'flags must be a contiguous ({env.N}, 4) uint8 tensor on {env.device}')


def as_command(env, dev, cmd):
    """`cmd` as a contiguous float32 tensor on the device `dev` of `env`, itself when it is one; ValueError unless it
    has shape (env.N, 2)"""
    a = cmd if (cmd.device == dev and cmd.dtype == torch.float32 and cmd.is_contiguous()) \
        else cmd.to(device=env.device, dtype=torch.float32).contiguous()
    if tuple(a.shape) != (env.N, 2):
        raise ValueError(f'the command must have shape ({env.N}, 2)')
    return a


def host_flags(flags, N):
    """Host flags as a contiguous (N, 4) uint8 array, or None; ValueError for another shape"""
    f = None if flags is None else np.ascontiguousarray(flags, np.uint8)
    if f is not None and f.shape != (N, 4):
        raise ValueError(f'flags must have shape ({N}, 4)')
    return f


def pair_argument(ap, args, flag, kind=float):
    """(a, b) of the command-line flag `flag` ('--scan-delay') given as A,B, or A for (A, A), each converted by `kind`;
    (0, 0) when it is not given.  ap.error naming the flag for anything else."""
    text = getattr(args, flag[2:].replace('-', '_'))
    if text is None:
        return kind(0), kind(0)
    parts = text.split(',')
    try:
        if len(parts) not in (1, 2):
            raise ValueError('takes one value or two separated by a comma')
        vals = [kind(p) for p in parts]
    except ValueError as e:
        ap.error('%s: %s' % (flag, e))
    return vals[0], vals[-1]
