"""Sensing and command latency around the tick (DESIGN.md §9q): the robots read the scan of d ticks earlier and
execute the command of l ticks earlier, with d and l drawn per robot for each episode, on the device by
csrc/rlca_latency.cu.

The tick and its outputs are never touched: `Latency.scan` replaces the newest frame of the caller's stack after a
tick, `Latency.action` writes the executed command into a buffer of its own before one.  The rings hold the true
frames and commands; env.obs, env.gs and the state stay the truth, so every tracker keeps measuring it.  A kind whose
range is (0, 0) allocates nothing and issues no launch.

    lat = Latency(env, LatencyParams(scan_delay=(1, 3), command_delay=(2, 2), seed=7))
    lat.scan(stacks[0])                             # the first stack: every row starts an episode
    executed = lat.action(scaled)                   # the first tick: no flags of a previous tick
    env.control_vel(executed, stack_in=stacks[0], stack_out=stacks[1])
    lat.scan(stacks[1], env.flags)                  # after the tick
    executed = lat.action(scaled, env.flags)        # every later tick: the flags of the tick before
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .perturbation import as_command, check_flags, check_seed, check_stack, check_stream_id, device_of, host_flags, \
    pair_argument, ptr

MAX_DELAY = 8                   # RLCA_LATENCY_MAX_DELAY: 0.8 s at dt = 0.1 s


def _delay_range(name, v):
    try:
        lo, hi = v
    except (TypeError, ValueError):
        raise ValueError(f'{name} must be a pair (lo, hi) of ticks, got {v!r}') from None
    for x in (lo, hi):
        if isinstance(x, bool) or int(x) != x:
            raise ValueError(f'{name} must hold whole ticks, got {v!r}')
    lo, hi = int(lo), int(hi)
    if not 0 <= lo <= hi <= MAX_DELAY:
        raise ValueError(f'{name} must satisfy 0 <= lo <= hi <= {MAX_DELAY} ticks, got ({lo}, {hi})')
    return lo, hi


@dataclass(frozen=True)
class LatencyParams:
    """scan_delay: (lo, hi) ticks the scan a robot reads is old; command_delay: (lo, hi) ticks between a command being
    issued and executed; each drawn uniformly per robot and episode, 0 <= lo <= hi <= MAX_DELAY.  seed: the Philox key
    of the draws (0 .. 2^64 - 1).  ValueError for anything else."""
    scan_delay: tuple = (0, 0)
    command_delay: tuple = (0, 0)
    seed: int = 0

    def __post_init__(self):
        object.__setattr__(self, 'scan_delay', _delay_range('scan_delay', self.scan_delay))
        object.__setattr__(self, 'command_delay', _delay_range('command_delay', self.command_delay))
        object.__setattr__(self, 'seed', check_seed('latency', self.seed))

    @property
    def scan_on(self):
        return self.scan_delay[1] > 0

    @property
    def command_on(self):
        return self.command_delay[1] > 0

    def as_dict(self):
        return {'scan_delay': list(self.scan_delay), 'command_delay': list(self.command_delay), 'seed': self.seed}

    def struct(self, stream_id=0):
        """_lib.LatencyParams of these settings for the env handle `stream_id`."""
        return _lib.LatencyParams(self.scan_delay[0], self.scan_delay[1], self.command_delay[0],
                                  self.command_delay[1], self.seed, check_stream_id(stream_id))


class Latency:
    """The latency of one env handle: its rings and per-robot delays.  `stream_id` tells apart the handles of one run
    (a mix component's index); the handle's world_offset tells apart the shards of a data-parallel run.  Every `scan`
    call and every `action` call advances its own counter by one; the counter picks the ring slot and the draw."""

    def __init__(self, env, params: LatencyParams, stream_id=0):
        if not isinstance(params, LatencyParams):
            raise TypeError('params must be a LatencyParams')
        self.env, self.params, self.stream_id = env, params, check_stream_id(stream_id)
        self._p = params.struct(self.stream_id)
        self._dev = device_of(env)
        N, B = env.N, env.beam_mum
        self.scan_calls = 0
        self.action_calls = 0
        self._scan_ring = self._scan_delay = self._cmd_ring = self._cmd_delay = self.executed = None
        if params.scan_on:
            self._scan_ring = torch.zeros(N, params.scan_delay[1] + 1, B, device=env.device)
            self._scan_delay = torch.zeros(N, dtype=torch.uint8, device=env.device)
        if params.command_on:
            self._cmd_ring = torch.zeros(N, params.command_delay[1] + 1, 2, device=env.device)
            self._cmd_delay = torch.zeros(N, dtype=torch.uint8, device=env.device)
            self.executed = torch.zeros(N, 2, device=env.device)
        self._state = _lib.LatencyState(*(t.data_ptr() if t is not None else None for t in
                                          (self._scan_ring, self._cmd_ring, self._scan_delay, self._cmd_delay)))

    def settings(self):
        return dict(self.params.as_dict(), stream_id=self.stream_id)

    @property
    def scan_delays(self):
        """(N,) uint8: the scan delay of each robot's current episode, ticks (a copy; zeros when scan delay is off)"""
        return self._scan_delay.clone() if self._scan_delay is not None else \
            torch.zeros(self.env.N, dtype=torch.uint8, device=self.env.device)

    @property
    def command_delays(self):
        """(N,) uint8: the command delay of each robot's current episode, ticks (a copy; zeros when off)"""
        return self._cmd_delay.clone() if self._cmd_delay is not None else \
            torch.zeros(self.env.N, dtype=torch.uint8, device=self.env.device)

    def scan(self, stack, flags=None):
        """After a tick (and any re-layout): replace the newest frame of `stack` (N, 3, beams) float32 in place with
        the frame of each robot's scan delay earlier, on the env's stream.  Rows whose flags[:, 3] (was_reset) is set,
        and every row when `flags` is None, start an episode: their delay is redrawn and their stack kept.  Returns
        `stack`."""
        env = self.env
        check_stack(env, self._dev, stack)
        check_flags(env, self._dev, flags)
        draw = self.scan_calls
        self.scan_calls += 1
        if self.params.scan_on:
            _lib.check(env.lib.rlca_latency_scan(C.byref(env.cfg), C.byref(self._p), C.byref(self._state),
                                                 draw & 0xFFFFFFFF, ptr(flags), ptr(stack), env._stream()))
        return stack

    def action(self, cmd, flags=None):
        """Before a tick: the command the robots execute for the issued command `cmd` (N, 2), which is not written.
        `flags` are those of the previous tick (None on a run's first tick): rows whose flags[:, 3] is set start an
        episode and execute its first command until l ticks have passed.  Returns `self.executed`, one buffer reused by every call, or `cmd` itself when
        command latency is off."""
        env = self.env
        check_flags(env, self._dev, flags)
        draw = self.action_calls
        self.action_calls += 1
        if not self.params.command_on:
            return cmd
        a = as_command(env, self._dev, cmd)
        _lib.check(env.lib.rlca_latency_action(C.byref(env.cfg), C.byref(self._p), C.byref(self._state),
                                               draw & 0xFFFFFFFF, ptr(flags), ptr(a), ptr(self.executed),
                                               env._stream()))
        return self.executed


class HostState:
    """Host rings and delays for scan_host / action_host: the same layout as Latency's device buffers."""

    def __init__(self, cfg, params: LatencyParams):
        N, B = int(cfg.robots_per_world) * int(cfg.num_worlds), int(cfg.beams)
        self.scan_ring = np.zeros((N, params.scan_delay[1] + 1, B), np.float32)
        self.cmd_ring = np.zeros((N, params.command_delay[1] + 1, 2), np.float32)
        self.scan_delay = np.zeros(N, np.uint8)
        self.cmd_delay = np.zeros(N, np.uint8)

    def struct(self):
        vp = lambda a: a.ctypes.data
        return _lib.LatencyState(vp(self.scan_ring), vp(self.cmd_ring), vp(self.scan_delay), vp(self.cmd_delay))


def scan_host(cfg, params: LatencyParams, state: HostState, draw, stack, flags=None, stream_id=0):
    """rlca_latency_scan_host on a host stack (N, 3, beams) float32, changed in place, and the HostState `state`
    (the kernel's code, run by the CPU); returns the stack."""
    N = int(cfg.robots_per_world) * int(cfg.num_worlds)
    if stack.dtype != np.float32 or not stack.flags.c_contiguous or stack.shape != (N, 3, int(cfg.beams)):
        raise ValueError(f'stack must be a contiguous ({N}, 3, {int(cfg.beams)}) float32 array')
    f = host_flags(flags, N)
    _lib.check(_lib.load().rlca_latency_scan_host(C.byref(cfg), C.byref(params.struct(stream_id)),
                                                  C.byref(state.struct()), int(draw),
                                                  f.ctypes.data_as(C.c_void_p) if f is not None else None,
                                                  stack.ctypes.data_as(C.c_void_p)))
    return stack


def action_host(cfg, params: LatencyParams, state: HostState, draw, cmd, flags=None, stream_id=0):
    """rlca_latency_action_host: the executed (N, 2) float32 command for the issued command `cmd` (not written)."""
    N = int(cfg.robots_per_world) * int(cfg.num_worlds)
    a = np.ascontiguousarray(cmd, np.float32)
    if a.shape != (N, 2):
        raise ValueError('cmd must have one (v, w) row per agent')
    f = host_flags(flags, N)
    out = np.empty_like(a)
    _lib.check(_lib.load().rlca_latency_action_host(C.byref(cfg), C.byref(params.struct(stream_id)),
                                                    C.byref(state.struct()), int(draw),
                                                    f.ctypes.data_as(C.c_void_p) if f is not None else None,
                                                    a.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
    return out


# ------------------------------------------------------------------------------------------------ command line
LATENCY_FLAGS = ('--scan-delay', '--command-delay', '--latency-seed')


def add_latency_arguments(ap):
    """The latency flags of a driver on an argparse parser; every one defaults to off."""
    ap.add_argument('--scan-delay', default=None, metavar='T[,T_MAX]',
                    help='the scan a robot reads is T ticks old (0.1 s each), or drawn in T..T_MAX per robot and '
                         'episode; at most %d (DESIGN.md §9q)' % MAX_DELAY)
    ap.add_argument('--command-delay', default=None, metavar='T[,T_MAX]',
                    help='a command is executed T ticks after it is issued, or T..T_MAX drawn per robot and episode')
    ap.add_argument('--latency-seed', type=int, default=None, metavar='S',
                    help='seed of the delay draws (default: --seed)')


def latency_from_arguments(ap, args):
    """LatencyParams of the latency flags, or None when none is given; ap.error for a bad value and for
    --latency-seed on its own.  The seed is --latency-seed, else --seed, else 0."""
    if args.scan_delay is None and args.command_delay is None:
        if args.latency_seed is not None:
            ap.error('--latency-seed applies with --scan-delay or --command-delay only')
        return None
    ranges = {name: pair_argument(ap, args, '--' + name.replace('_', '-'), int)
              for name in ('scan_delay', 'command_delay')}
    seed = args.latency_seed if args.latency_seed is not None else getattr(args, 'seed', 0)
    try:
        return LatencyParams(seed=seed, **ranges)
    except ValueError as e:
        ap.error('latency: %s' % e)
