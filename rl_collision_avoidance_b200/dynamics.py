"""Acceleration limits just before the tick (DESIGN.md §9r): each robot's v and w move from the velocity it executed on
the last tick towards its command by at most a dt and b dt, with the linear limit a and the angular limit b drawn per
robot for each episode, on the device by csrc/rlca_dynamics.cu.

The tick and its outputs are never touched: `Dynamics.action` writes the executed command into a buffer of its own
before a tick, and keeps the executed velocity as its own state.  env.obs, env.gs and the state stay what the tick
made them, so every tracker keeps measuring them.  The tick writes the executed command into gs, so the speed a
policy reads is the limited one, as odometry would report it.

    dyn = Dynamics(env, DynamicsParams(linear=(1.0, 1.0), angular=(1.0, 4.0), seed=7))
    executed = dyn.action(scaled)                   # the first tick: every robot starts from rest
    env.control_vel(executed, stack_in=stacks[0], stack_out=stacks[1])
    executed = dyn.action(scaled, env.flags)        # every later tick: the flags of the tick before
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .latency import _host_flags, _ptr, check_flags
from .noise import check_stream_id

MAX_ACCEL = 100.0               # RLCA_DYNAMICS_MAX_ACCEL, m/s^2 and rad/s^2


def _accel_range(name, v):
    """(lo, hi) as the float32 values the kernel uses: (0, 0), or finite with 0 < lo <= hi <= MAX_ACCEL"""
    try:
        lo, hi = v
    except (TypeError, ValueError):
        raise ValueError(f'{name} must be a pair (lo, hi), got {v!r}') from None
    if isinstance(lo, bool) or isinstance(hi, bool):
        raise ValueError(f'{name} must hold numbers, got {v!r}')
    lo, hi = float(np.float32(lo)), float(np.float32(hi))
    if not ((lo == 0.0 and hi == 0.0) or (math.isfinite(hi) and 0.0 < lo <= hi <= MAX_ACCEL)):
        raise ValueError(f'{name} must be (0, 0) (off) or satisfy 0 < lo <= hi <= {MAX_ACCEL:g}, got {v!r}')
    return lo, hi


@dataclass(frozen=True)
class DynamicsParams:
    """linear: (lo, hi) m/s^2 of the linear acceleration limit, angular: (lo, hi) rad/s^2 of the angular one; each drawn
    uniformly per robot and episode, (0, 0) for a kind that is off, else 0 < lo <= hi <= MAX_ACCEL (held as float32).
    seed: the Philox key of the draws (0 .. 2^64 - 1).  ValueError for anything else."""
    linear: tuple = (0.0, 0.0)
    angular: tuple = (0.0, 0.0)
    seed: int = 0

    def __post_init__(self):
        object.__setattr__(self, 'linear', _accel_range('linear', self.linear))
        object.__setattr__(self, 'angular', _accel_range('angular', self.angular))
        if isinstance(self.seed, bool) or int(self.seed) != self.seed or not 0 <= int(self.seed) < 1 << 64:
            raise ValueError(f'the dynamics seed must be an integer in 0 .. 2^64 - 1, got {self.seed!r}')
        object.__setattr__(self, 'seed', int(self.seed))

    @property
    def linear_on(self):
        return self.linear[1] > 0.0

    @property
    def angular_on(self):
        return self.angular[1] > 0.0

    def as_dict(self):
        return {'linear': list(self.linear), 'angular': list(self.angular), 'seed': self.seed}

    def struct(self, stream_id=0):
        """_lib.DynamicsParams of these settings for the env handle `stream_id`."""
        return _lib.DynamicsParams(self.linear[0], self.linear[1], self.angular[0], self.angular[1], self.seed,
                                   check_stream_id(stream_id))


class Dynamics:
    """The acceleration limits of one env handle: each robot's executed velocity and its limits.  `stream_id` tells
    apart the handles of one run (a mix component's index); the handle's world_offset tells apart the shards of a
    data-parallel run.  Every `action` call advances the draw counter by one."""

    def __init__(self, env, params: DynamicsParams, stream_id=0):
        if not isinstance(params, DynamicsParams):
            raise TypeError('params must be a DynamicsParams')
        self.env, self.params, self.stream_id = env, params, check_stream_id(stream_id)
        self._p = params.struct(self.stream_id)
        d = torch.device(env.device)
        self._dev = d if d.index is not None or d.type != 'cuda' else torch.device('cuda', torch.cuda.current_device())
        N = env.N
        self.calls = 0
        self._vel = torch.zeros(N, 2, device=env.device)
        self._lin = torch.zeros(N, device=env.device)
        self._ang = torch.zeros(N, device=env.device)
        self.executed = torch.zeros(N, 2, device=env.device)
        self._state = _lib.DynamicsState(self._vel.data_ptr(), self._lin.data_ptr(), self._ang.data_ptr())

    def settings(self):
        return dict(self.params.as_dict(), stream_id=self.stream_id)

    @property
    def limits(self):
        """(N, 2) float32: the linear (m/s^2) and angular (rad/s^2) limit of each robot's current episode (a copy; 0
        for a kind that is off)"""
        return torch.stack((self._lin, self._ang), 1)

    def action(self, cmd, flags=None):
        """Before a tick: the command the robots execute for the command `cmd` (N, 2), which is not written.  `flags`
        are those of the previous tick (None on a run's first tick): rows whose flags[:, 3] (was_reset) is set start an
        episode, draw their limits and start from rest; rows whose flags[:, 1] (crashed) is set start from rest.
        Returns `self.executed`, one buffer reused by every call."""
        env = self.env
        check_flags(env, self._dev, flags)
        a = cmd if (cmd.device == self._dev and cmd.dtype == torch.float32 and cmd.is_contiguous()) \
            else cmd.to(device=env.device, dtype=torch.float32).contiguous()
        if tuple(a.shape) != (env.N, 2):
            raise ValueError(f'the command must have shape ({env.N}, 2)')
        draw = self.calls
        self.calls += 1
        _lib.check(env.lib.rlca_dynamics_action(C.byref(env.cfg), C.byref(self._p), C.byref(self._state),
                                                draw & 0xFFFFFFFF, _ptr(flags), _ptr(a), _ptr(self.executed),
                                                env._stream()))
        return self.executed


class HostState:
    """Host velocity and limits for action_host: the same layout as Dynamics' device buffers."""

    def __init__(self, cfg):
        N = int(cfg.robots_per_world) * int(cfg.num_worlds)
        self.vel = np.zeros((N, 2), np.float32)
        self.lin_limit = np.zeros(N, np.float32)
        self.ang_limit = np.zeros(N, np.float32)

    def struct(self):
        return _lib.DynamicsState(self.vel.ctypes.data, self.lin_limit.ctypes.data, self.ang_limit.ctypes.data)


def action_host(cfg, params: DynamicsParams, state: HostState, draw, cmd, flags=None, stream_id=0):
    """rlca_dynamics_action_host: the executed (N, 2) float32 command for the command `cmd` (not written), with the
    HostState `state` updated (the kernel's code, run by the CPU)."""
    N = int(cfg.robots_per_world) * int(cfg.num_worlds)
    a = np.ascontiguousarray(cmd, np.float32)
    if a.shape != (N, 2):
        raise ValueError('cmd must have one (v, w) row per agent')
    f = _host_flags(flags, N)
    out = np.empty_like(a)
    _lib.check(_lib.load().rlca_dynamics_action_host(C.byref(cfg), C.byref(params.struct(stream_id)),
                                                     C.byref(state.struct()), int(draw),
                                                     f.ctypes.data_as(C.c_void_p) if f is not None else None,
                                                     a.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
    return out


# ------------------------------------------------------------------------------------------------ command line
DYNAMICS_FLAGS = ('--accel-limit', '--angular-accel-limit', '--dynamics-seed')


def add_dynamics_arguments(ap):
    """The acceleration-limit flags of a driver on an argparse parser; every one defaults to off."""
    ap.add_argument('--accel-limit', default=None, metavar='A[,A_MAX]',
                    help='linear acceleration limit, m/s^2, or drawn in A..A_MAX per robot and episode; in (0, %g] '
                         '(DESIGN.md §9r)' % MAX_ACCEL)
    ap.add_argument('--angular-accel-limit', default=None, metavar='B[,B_MAX]',
                    help='angular acceleration limit, rad/s^2, or drawn in B..B_MAX per robot and episode')
    ap.add_argument('--dynamics-seed', type=int, default=None, metavar='S',
                    help='seed of the limit draws (default: --seed)')


def _limits(text):
    parts = text.split(',')
    if len(parts) not in (1, 2):
        raise ValueError('takes A or A,A_MAX')
    vals = [float(p) for p in parts]
    return (vals[0], vals[0]) if len(vals) == 1 else tuple(vals)


def dynamics_from_arguments(ap, args):
    """DynamicsParams of the acceleration-limit flags, or None when none is given; ap.error for a bad value (a limit
    of 0 included: leave the flag out instead) and for --dynamics-seed on its own.  The seed is --dynamics-seed, else
    --seed, else 0."""
    if args.accel_limit is None and args.angular_accel_limit is None:
        if args.dynamics_seed is not None:
            ap.error('--dynamics-seed applies with --accel-limit or --angular-accel-limit only')
        return None
    ranges = {}
    for name, flag in (('linear', 'accel_limit'), ('angular', 'angular_accel_limit')):
        text = getattr(args, flag)
        try:
            ranges[name] = _limits(text) if text is not None else (0.0, 0.0)
        except ValueError as e:
            ap.error('--%s: %s' % (flag.replace('_', '-'), e))
        if text is not None and ranges[name][0] <= 0.0:
            ap.error('--%s: a limit must be > 0' % flag.replace('_', '-'))
    seed = args.dynamics_seed if args.dynamics_seed is not None else getattr(args, 'seed', 0)
    try:
        return DynamicsParams(seed=seed, **ranges)
    except ValueError as e:
        ap.error('dynamics: %s' % e)
