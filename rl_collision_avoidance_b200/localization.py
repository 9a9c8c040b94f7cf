"""Localization error in the policy's goal and speed inputs (DESIGN.md §9s): each robot's local goal is computed from a
believed pose (x + ex, y + ey, theta + etheta) whose error follows a Gauss-Markov process per robot, and its speed reads
with white odometry noise, drawn on the device by csrc/rlca_localization.cu.

The tick and its outputs are never touched: `Localization.observe` writes the believed gs into a buffer of its own (or
the caller's) after a tick, and keeps the error as its own state.  env.obs, env.gs and the state stay the truth, so
success, crashes, rewards and every tracker keep measuring it.  Settings that are all zero allocate nothing and issue
no launch.

    loc = Localization(env, LocalizationParams(pose_sigma=(0.1, 0.3), heading_sigma=(0.05, 0.05),
                                               correlation_time=2.0, speed_sigma=(0.05, 0.1), seed=7))
    gs = loc.observe()                              # the first gs: every robot starts an episode
    env.control_vel(executed, stack_in=stacks[0], stack_out=stacks[1])
    gs = loc.observe(env.flags)                     # after every tick: the flags of that tick
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .perturbation import check_flags, check_seed, check_stream_id, device_of, host_flags, pair_argument, ptr

DEFAULT_CORRELATION_TIME = 2.0  # s


def _sigma_pair(name, v, ordered=True):
    """(a, b) as the float32 values the kernel uses: finite, >= 0, and a <= b when `ordered` (a range)"""
    try:
        lo, hi = v
    except (TypeError, ValueError):
        raise ValueError(f'{name} must be a pair, got {v!r}') from None
    if isinstance(lo, bool) or isinstance(hi, bool):
        raise ValueError(f'{name} must hold numbers, got {v!r}')
    with np.errstate(over='ignore'):                 # a value beyond float32 becomes inf and is refused below
        lo, hi = float(np.float32(lo)), float(np.float32(hi))
    if not (math.isfinite(lo) and math.isfinite(hi) and lo >= 0.0 and hi >= 0.0 and (lo <= hi or not ordered)):
        raise ValueError(f'{name} must be finite and >= 0' + (' with lo <= hi' if ordered else '') + f', got {v!r}')
    return lo, hi


@dataclass(frozen=True)
class LocalizationParams:
    """pose_sigma: (lo, hi) m of the standard deviation of ex and ey, heading_sigma: (lo, hi) rad of etheta's, each
    drawn uniformly per robot and episode; correlation_time: tau, s, of the Gauss-Markov error (0 white jitter on every
    tick, inf a constant offset for the episode); speed_sigma: (sigma_v m/s, sigma_w rad/s) of the white noise on the
    speed the policy reads.  Every value is held as float32; sigmas finite and >= 0, tau >= 0 or inf.  seed: the Philox
    key of the draws (0 .. 2^64 - 1).  ValueError for anything else."""
    pose_sigma: tuple = (0.0, 0.0)
    heading_sigma: tuple = (0.0, 0.0)
    correlation_time: float = DEFAULT_CORRELATION_TIME
    speed_sigma: tuple = (0.0, 0.0)
    seed: int = 0

    def __post_init__(self):
        object.__setattr__(self, 'pose_sigma', _sigma_pair('pose_sigma', self.pose_sigma))
        object.__setattr__(self, 'heading_sigma', _sigma_pair('heading_sigma', self.heading_sigma))
        object.__setattr__(self, 'speed_sigma', _sigma_pair('speed_sigma', self.speed_sigma, ordered=False))
        tau = self.correlation_time
        if isinstance(tau, bool) or not isinstance(tau, (int, float, np.floating, np.integer)):
            raise ValueError(f'correlation_time must be a number, got {tau!r}')
        tau = float(np.float32(tau))
        if not tau >= 0.0:
            raise ValueError(f'correlation_time must be >= 0 s or inf, got {self.correlation_time!r}')
        object.__setattr__(self, 'correlation_time', tau)
        object.__setattr__(self, 'seed', check_seed('localization', self.seed))

    @property
    def on(self):
        return self.pose_sigma[1] > 0.0 or self.heading_sigma[1] > 0.0 or self.speed_sigma[0] > 0.0 or \
            self.speed_sigma[1] > 0.0

    def as_dict(self):
        return {'pose_sigma': list(self.pose_sigma), 'heading_sigma': list(self.heading_sigma),
                'correlation_time': self.correlation_time, 'speed_sigma': list(self.speed_sigma), 'seed': self.seed}

    def struct(self, stream_id=0):
        """_lib.LocalizationParams of these settings for the env handle `stream_id`."""
        return _lib.LocalizationParams(self.pose_sigma[0], self.pose_sigma[1], self.heading_sigma[0],
                                       self.heading_sigma[1], self.correlation_time, self.speed_sigma[0],
                                       self.speed_sigma[1], self.seed, check_stream_id(stream_id))


class Localization:
    """The localization error of one env handle: each robot's pose-estimate error and its standard deviations.
    `stream_id` tells apart the handles of one run (a mix component's index); the handle's world_offset tells apart the
    shards of a data-parallel run.  Every `observe` call advances the draw counter by one."""

    def __init__(self, env, params: LocalizationParams, stream_id=0):
        if not isinstance(params, LocalizationParams):
            raise TypeError('params must be a LocalizationParams')
        self.env, self.params, self.stream_id = env, params, check_stream_id(stream_id)
        self._p = params.struct(self.stream_id)
        self._dev = device_of(env)
        self.calls = 0
        self._err = self._sigma = self.believed = None
        if params.on:
            N = env.N
            self._err = torch.zeros(N, 4, device=env.device)
            self._sigma = torch.zeros(N, 2, device=env.device)
            self.believed = torch.zeros(N, 4, device=env.device)
            self._state = _lib.LocalizationState(self._err.data_ptr(), self._sigma.data_ptr())

    def settings(self):
        return dict(self.params.as_dict(), stream_id=self.stream_id)

    @property
    def errors(self):
        """(N, 3) float32: ex, ey (m) and etheta (rad) of each robot's current pose estimate (a copy; 0 when off)"""
        return self._err[:, 0:3].clone() if self._err is not None else \
            torch.zeros(self.env.N, 3, device=self.env.device)

    @property
    def sigmas(self):
        """(N, 2) float32: sigma_xy (m) and sigma_theta (rad) of each robot's current episode (a copy; 0 when off)"""
        return self._sigma.clone() if self._sigma is not None else torch.zeros(self.env.N, 2, device=self.env.device)

    def _check_gs(self, name, t):
        env = self.env
        if tuple(t.shape) != (env.N, 4) or t.dtype != torch.float32 or not t.is_contiguous() or t.device != self._dev:
            raise ValueError(f'{name} must be a contiguous ({env.N}, 4) float32 tensor on {env.device}')

    def observe(self, flags=None, gs=None, out=None):
        """After a tick (and any re-layout, latency and noise): the gs (N, 4) the policy reads, from the true `gs`
        (default env.gs, never written unless it is `out`) and the env's current state.  `flags` are those of the tick
        just run (None for a run's first gs): rows whose flags[:, 3] (was_reset) is set start an episode, draw their
        sigmas and a fresh error.  Writes `out` (default `self.believed`, one buffer reused by every call; `gs` itself
        for in place) and returns it; with settings that are all zero nothing is launched and `gs` is returned (copied
        into `out` when one is given)."""
        env = self.env
        check_flags(env, self._dev, flags)
        g = env.gs if gs is None else gs
        self._check_gs('gs', g)
        if out is not None:
            self._check_gs('out', out)
        draw = self.calls
        self.calls += 1
        if not self.params.on:
            if out is None or out.data_ptr() == g.data_ptr():
                return g
            return out.copy_(g)
        o = self.believed if out is None else out
        _lib.check(env.lib.rlca_localization_observe(C.byref(env.cfg), C.byref(self._p), C.byref(self._state),
                                                     draw & 0xFFFFFFFF, ptr(flags),
                                                     C.byref(env._state_struct(env._cur)), ptr(g), ptr(o),
                                                     env._stream()))
        return o


class HostState:
    """Host error and sigmas for observe_host: the same layout as Localization's device buffers."""

    def __init__(self, cfg):
        N = int(cfg.robots_per_world) * int(cfg.num_worlds)
        self.err = np.zeros((N, 4), np.float32)
        self.sigma = np.zeros((N, 2), np.float32)

    def struct(self):
        return _lib.LocalizationState(self.err.ctypes.data, self.sigma.ctypes.data)


def observe_host(cfg, params: LocalizationParams, state: HostState, draw, pose, goal, gs, flags=None, stream_id=0):
    """rlca_localization_observe_host: the believed (N, 4) float32 gs from the env state's `pose` and `goal` (N, 4) and
    the true `gs` (N, 4), none of them written, with the HostState `state` updated (the kernel's code, run by the
    CPU)."""
    N = int(cfg.robots_per_world) * int(cfg.num_worlds)
    arrs = []
    for name, a in (('pose', pose), ('goal', goal), ('gs', gs)):
        a = np.ascontiguousarray(a, np.float32)
        if a.shape != (N, 4):
            raise ValueError(f'{name} must have one row of 4 per agent')
        arrs.append(a)
    p, g, s = arrs
    f = host_flags(flags, N)
    out = np.empty_like(s)
    st = _lib.EnvState(p.ctypes.data, g.ctypes.data, None, None)
    _lib.check(_lib.load().rlca_localization_observe_host(C.byref(cfg), C.byref(params.struct(stream_id)),
                                                          C.byref(state.struct()), int(draw),
                                                          f.ctypes.data_as(C.c_void_p) if f is not None else None,
                                                          C.byref(st), s.ctypes.data_as(C.c_void_p),
                                                          out.ctypes.data_as(C.c_void_p)))
    return out


# ------------------------------------------------------------------------------------------------ command line
LOCALIZATION_FLAGS = ('--pose-error', '--heading-error', '--pose-error-time', '--speed-error', '--localization-seed')


def add_localization_arguments(ap):
    """The localization-error flags of a driver on an argparse parser; every one defaults to off."""
    ap.add_argument('--pose-error', default=None, metavar='S[,S_MAX]',
                    help='standard deviation of the position error of the pose the local goal is computed from, m, or '
                         'drawn in S..S_MAX per robot and episode (DESIGN.md §9s)')
    ap.add_argument('--heading-error', default=None, metavar='S[,S_MAX]',
                    help='standard deviation of the heading error of that pose, rad, or drawn in S..S_MAX')
    ap.add_argument('--pose-error-time', type=float, default=None, metavar='T',
                    help='correlation time of the pose and heading error, s: 0 new on every tick, inf one offset per '
                         'episode (default %g)' % DEFAULT_CORRELATION_TIME)
    ap.add_argument('--speed-error', default=None, metavar='SV[,SW]',
                    help='white noise on the speed the policy reads: N(0, SV^2) m/s on v and N(0, SW^2) rad/s on w; '
                         'one value sets both')
    ap.add_argument('--localization-seed', type=int, default=None, metavar='S',
                    help='seed of the localization draws (default: --seed)')


def localization_from_arguments(ap, args):
    """LocalizationParams of the localization flags, or None when none is given; ap.error for a bad value, for
    --pose-error-time without --pose-error or --heading-error and for --localization-seed on its own.  The seed is
    --localization-seed, else --seed, else 0."""
    pose_time = args.pose_error_time is not None
    if pose_time and args.pose_error is None and args.heading_error is None:
        ap.error('--pose-error-time applies with --pose-error or --heading-error only')
    if args.pose_error is None and args.heading_error is None and args.speed_error is None:
        if args.localization_seed is not None:
            ap.error('--localization-seed applies with --pose-error, --heading-error or --speed-error only')
        return None
    vals = {name: pair_argument(ap, args, flag) for name, flag in
            (('pose_sigma', '--pose-error'), ('heading_sigma', '--heading-error'), ('speed_sigma', '--speed-error'))}
    seed = args.localization_seed if args.localization_seed is not None else getattr(args, 'seed', 0)
    tau = args.pose_error_time if pose_time else DEFAULT_CORRELATION_TIME
    try:
        return LocalizationParams(correlation_time=tau, seed=seed, **vals)
    except ValueError as e:
        ap.error('localization: %s' % e)
