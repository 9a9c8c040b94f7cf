"""Sensor and actuation noise around the tick (DESIGN.md §9p): lidar range noise and beam dropout on the newest frame of
an observation stack, and a gain error on the executed (v, w), drawn on the device by csrc/rlca_noise.cu.

The tick and its outputs are never touched: `Noise.scan` perturbs the caller's stack after a tick, `Noise.action`
writes the executed command into a buffer of its own before one.  Settings that are all zero issue no launch at all.

    noise = Noise(env, NoiseParams(range_sigma=0.05, dropout=0.1, v_gain_sigma=0.1, w_gain_sigma=0.1, seed=7))
    noise.scan(stacks[0])                           # the first stack: every row fresh
    executed = noise.action(scaled)                 # before the tick; `scaled` is not written
    env.control_vel(executed, stack_in=stacks[0], stack_out=stacks[1])
    noise.scan(stacks[1], env.flags)                # after the tick
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import asdict, dataclass

import numpy as np
import torch

from . import _lib

MAX_STREAM_ID = (1 << 24) - 1


def _finite_nonneg(name, v):
    v = float(v)
    if not (math.isfinite(v) and v >= 0.0):
        raise ValueError(f'{name} must be finite and >= 0, got {v!r}')
    return v


@dataclass(frozen=True)
class NoiseParams:
    """range_sigma: standard deviation of the range error of a beam with a return, metres; dropout: probability that a
    beam reads no return; v_gain_sigma, w_gain_sigma: standard deviation of the relative gain error of the executed v
    and w; seed: the Philox key of every draw (0 .. 2^64 - 1).  ValueError for anything else."""
    range_sigma: float = 0.0
    dropout: float = 0.0
    v_gain_sigma: float = 0.0
    w_gain_sigma: float = 0.0
    seed: int = 0

    def __post_init__(self):
        for k in ('range_sigma', 'v_gain_sigma', 'w_gain_sigma'):
            object.__setattr__(self, k, _finite_nonneg(k, getattr(self, k)))
        p = float(self.dropout)
        if not 0.0 <= p <= 1.0:
            raise ValueError(f'dropout must be in [0, 1], got {self.dropout!r}')
        object.__setattr__(self, 'dropout', p)
        if isinstance(self.seed, bool) or int(self.seed) != self.seed or not 0 <= int(self.seed) < 1 << 64:
            raise ValueError(f'the noise seed must be an integer in 0 .. 2^64 - 1, got {self.seed!r}')
        object.__setattr__(self, 'seed', int(self.seed))

    @property
    def scan_on(self):
        return self.range_sigma > 0.0 or self.dropout > 0.0

    @property
    def action_on(self):
        return self.v_gain_sigma > 0.0 or self.w_gain_sigma > 0.0

    def as_dict(self):
        return asdict(self)

    def struct(self, stream_id=0):
        """_lib.NoiseParams of these settings for the env handle `stream_id`."""
        return _lib.NoiseParams(self.range_sigma, self.dropout, self.v_gain_sigma, self.w_gain_sigma, self.seed,
                                check_stream_id(stream_id))


def check_stream_id(stream_id):
    if isinstance(stream_id, bool) or int(stream_id) != stream_id or not 0 <= int(stream_id) <= MAX_STREAM_ID:
        raise ValueError(f'stream_id must be an integer in 0 .. {MAX_STREAM_ID}, got {stream_id!r}')
    return int(stream_id)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class Noise:
    """The noise of one env handle.  `stream_id` tells apart the handles of one run (a mix component's index), so that
    agent 0 of two handles draws different noise; the handle's world_offset tells apart the shards of a data-parallel
    run.  Every `scan` call and every `action` call advances its own draw counter by one."""

    def __init__(self, env, params: NoiseParams, stream_id=0):
        if not isinstance(params, NoiseParams):
            raise TypeError('params must be a NoiseParams')
        self.env, self.params, self.stream_id = env, params, check_stream_id(stream_id)
        self._p = params.struct(self.stream_id)
        d = torch.device(env.device)
        self._dev = d if d.index is not None or d.type != 'cuda' else torch.device('cuda', torch.cuda.current_device())
        self.scan_draws = 0
        self.action_draws = 0
        self.executed = torch.zeros(env.N, 2, device=env.device) if params.action_on else None

    def settings(self):
        return dict(self.params.as_dict(), stream_id=self.stream_id)

    def scan(self, stack, flags=None):
        """Perturb the newest frame of `stack` (N, 3, beams) float32 in place, on the env's stream.  Rows whose
        flags[:, 3] (was_reset) is set, and every row when `flags` is None, get the perturbed frame in all three
        slots.  Returns `stack`."""
        env = self.env
        if tuple(stack.shape) != (env.N, 3, env.beam_mum) or stack.dtype != torch.float32 or \
                not stack.is_contiguous() or stack.device != self._dev:
            raise ValueError(f'stack must be a contiguous ({env.N}, 3, {env.beam_mum}) float32 tensor on {env.device}')
        if flags is not None and (tuple(flags.shape) != (env.N, 4) or flags.dtype != torch.uint8 or
                                  not flags.is_contiguous() or flags.device != self._dev):
            raise ValueError(f'flags must be a contiguous ({env.N}, 4) uint8 tensor on {env.device}')
        draw = self.scan_draws
        self.scan_draws += 1
        if self.params.scan_on:
            _lib.check(env.lib.rlca_noise_scan(C.byref(env.cfg), C.byref(self._p), draw & 0xFFFFFFFF, _ptr(flags),
                                               _ptr(stack), env._stream()))
        return stack

    def action(self, scaled):
        """The command the robots execute for the command `scaled` (N, 2), which is not written: `self.executed`, one
        buffer reused by every call, or `scaled` itself when the settings have no actuation noise."""
        env = self.env
        draw = self.action_draws
        self.action_draws += 1
        if not self.params.action_on:
            return scaled
        a = scaled if (scaled.device == self._dev and scaled.dtype == torch.float32 and scaled.is_contiguous()) \
            else scaled.to(device=env.device, dtype=torch.float32).contiguous()
        if tuple(a.shape) != (env.N, 2):
            raise ValueError(f'the command must have shape ({env.N}, 2)')
        _lib.check(env.lib.rlca_noise_action(C.byref(env.cfg), C.byref(self._p), draw & 0xFFFFFFFF, _ptr(a),
                                             _ptr(self.executed), env._stream()))
        return self.executed


def scan_host(cfg, params: NoiseParams, draw, stack, flags=None, stream_id=0):
    """rlca_noise_scan_host on a host stack (N, 3, beams) float32, perturbed in place (the kernel's code, run by the
    CPU); returns it."""
    N = int(cfg.robots_per_world) * int(cfg.num_worlds)
    if stack.dtype != np.float32 or not stack.flags.c_contiguous or stack.shape != (N, 3, int(cfg.beams)):
        raise ValueError(f'stack must be a contiguous ({N}, 3, {int(cfg.beams)}) float32 array')
    f = None if flags is None else np.ascontiguousarray(flags, np.uint8)
    if f is not None and f.shape != (N, 4):
        raise ValueError(f'flags must have shape ({N}, 4)')
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    _lib.check(_lib.load().rlca_noise_scan_host(C.byref(cfg), C.byref(params.struct(stream_id)), int(draw), vp(f),
                                                vp(stack)))
    return stack


def action_host(cfg, params: NoiseParams, draw, action, stream_id=0):
    """rlca_noise_action_host: the executed (N, 2) float32 command for the command `action` (not written)."""
    a = np.ascontiguousarray(action, np.float32)
    if a.shape != (int(cfg.robots_per_world) * int(cfg.num_worlds), 2):
        raise ValueError('action must have one (v, w) row per agent')
    out = np.empty_like(a)
    _lib.check(_lib.load().rlca_noise_action_host(C.byref(cfg), C.byref(params.struct(stream_id)), int(draw),
                                                  a.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
    return out


# ------------------------------------------------------------------------------------------------ command line
NOISE_FLAGS = ('--scan-noise', '--beam-dropout', '--action-noise', '--noise-seed')


def add_noise_arguments(ap):
    """The noise flags of a driver on an argparse parser; every one defaults to off."""
    ap.add_argument('--scan-noise', type=float, default=None, metavar='SIGMA_M',
                    help='lidar range noise: a beam with a return reads r + N(0, SIGMA_M^2) m, clamped to [0, range_max] '
                         '(DESIGN.md §9p)')
    ap.add_argument('--beam-dropout', type=float, default=None, metavar='P',
                    help='each beam of each scan reads no return with probability P')
    ap.add_argument('--action-noise', default=None, metavar='SIGMA_V[,SIGMA_W]',
                    help='actuation noise: the executed v and w are the command times 1 + N(0, SIGMA^2) (at least 0), '
                         'clipped to the action bound; one value sets both')
    ap.add_argument('--noise-seed', type=int, default=None, metavar='S',
                    help='seed of the noise draws (default: --seed)')


def _action_sigmas(text):
    parts = text.split(',')
    if len(parts) not in (1, 2):
        raise ValueError('--action-noise takes SIGMA or SIGMA_V,SIGMA_W')
    vals = [float(p) for p in parts]
    return (vals[0], vals[0]) if len(vals) == 1 else tuple(vals)


def noise_from_arguments(ap, args):
    """NoiseParams of the noise flags, or None when none is given; ap.error for a bad value and for --noise-seed on its
    own.  The seed is --noise-seed, else --seed, else 0."""
    given = [getattr(args, f[2:].replace('-', '_')) is not None for f in NOISE_FLAGS[:3]]
    if not any(given):
        if args.noise_seed is not None:
            ap.error('--noise-seed applies with --scan-noise, --beam-dropout or --action-noise only')
        return None
    try:
        sv, sw = _action_sigmas(args.action_noise) if args.action_noise is not None else (0.0, 0.0)
    except ValueError as e:
        ap.error('--action-noise: %s' % e)
    seed = args.noise_seed if args.noise_seed is not None else getattr(args, 'seed', 0)
    try:
        return NoiseParams(range_sigma=args.scan_noise if args.scan_noise is not None else 0.0,
                           dropout=args.beam_dropout if args.beam_dropout is not None else 0.0,
                           v_gain_sigma=sv, w_gain_sigma=sw, seed=seed)
    except ValueError as e:
        ap.error('noise: %s' % e)
