"""The dynamic-window baseline (DESIGN.md §9u): a sensor-level classical controller on the device
(csrc/rlca_dwa.cu, rlca_dwa_action) that reads exactly what the policy reads: the newest frame of the scan stack, the
local goal and the robot's own speed.  It can therefore stand in the policy's slot of evaluate(), where scan noise,
beam dropout, scan delay and localization error apply to it as they do to the policy.

    dwa = DwaController(env, DwaParams())
    action = dwa(stack, gs)                 # (N, 2), one buffer reused by every call; dwa.status() per robot

`dwa_host` runs the same code on the CPU from numpy arrays and equals the kernel bit for bit.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import asdict, dataclass

import numpy as np
import torch

from . import _lib

MAX_CANDIDATES = 1024       # RLCA_DWA_MAX_CANDIDATES (include/rlca.h)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


@dataclass(frozen=True)
class DwaParams:
    """The dynamic-window settings (DESIGN.md §9u): starting values, not tuned ones.  ValueError for a value the kernel
    refuses."""
    v_samples: int = 11
    w_samples: int = 21
    radius: float = 0.30            # m: the footprint's 0.2907 m circumradius rounded up, as NH-ORCA's
    horizon: float = 2.0            # s
    heading_time: float = 1.0       # s
    accel: float = 0.0              # m/s^2, 0 = the whole action box (the simulator executes a command at once)
    angular_accel: float = 0.0      # rad/s^2, the same
    brake: float = 1.0              # m/s^2
    heading_weight: float = 1.0
    clearance_weight: float = 0.2
    speed_weight: float = 0.2
    clearance_cap: float = 1.0      # m (v_max * horizon froze the robots beside their goals: DESIGN.md §9u)

    def __post_init__(self):
        for k in ('v_samples', 'w_samples'):
            v = getattr(self, k)
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
                raise ValueError(f'dwa {k} must be an integer >= 1, got {v!r}')
        if self.v_samples * self.w_samples > MAX_CANDIDATES:
            raise ValueError(f'dwa v_samples * w_samples must be at most {MAX_CANDIDATES}, got '
                             f'{self.v_samples * self.w_samples}')

        def fin(k):
            v = getattr(self, k)
            if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)):
                raise ValueError(f'dwa {k} must be a number, got {v!r}')
            return float(v)
        for k in ('radius', 'horizon', 'brake', 'clearance_cap'):
            if not (math.isfinite(fin(k)) and fin(k) > 0.0):
                raise ValueError(f'dwa {k} must be finite and > 0, got {getattr(self, k)!r}')
        for k in ('heading_time', 'accel', 'angular_accel', 'heading_weight', 'clearance_weight', 'speed_weight'):
            if not (math.isfinite(fin(k)) and fin(k) >= 0.0):
                raise ValueError(f'dwa {k} must be finite and >= 0, got {getattr(self, k)!r}')

    def struct(self):
        """The rlca_dwa_params of these settings."""
        return _lib.DwaParams(**asdict(self))


def beam_directions(cfg):
    """(beams, 2) float32 unit vectors (cos b, sin b) of every beam in the robot frame, b measured from the heading:
    the env's own observation index map (the nearest-index sub-sampling of the raw beams, identity when beams =
    raw_beams), each evaluated in double and rounded to float as the env's beam table is."""
    raw, nb = int(cfg.raw_beams), int(cfg.beams)
    step, half = raw / nb, nb // 2
    idx = np.zeros(nb, np.int64)
    index = 0.0
    for i in range(half):
        idx[i] = int(index)
        index += step
    index = raw - 1.0
    for i in range(half):
        idx[nb - 1 - i] = int(index)
        index -= step
    fov = float(np.float32(cfg.fov))
    b = -0.5 * fov + idx.astype(np.float64) * (fov / (raw - 1))
    return np.ascontiguousarray(np.stack((np.cos(b), np.sin(b)), 1).astype(np.float32))


class DwaController:
    """The dynamic-window baseline on every robot of a StageWorld (rlca_dwa_action).  Calling it with the scan stack
    (N, 3, beams) and gs (N, 4) the policy would read (float32, contiguous, on the env's device) returns the (N, 2)
    command, written on the env's stream into one buffer that every call reuses."""

    def __init__(self, env, params=None):
        self.env = env
        self.params = DwaParams() if params is None else params
        self._p = self.params.struct()
        N, dev = env.N, env.device
        self.directions = torch.from_numpy(beam_directions(env.cfg)).to(dev)
        self.action = torch.zeros(N, 2, device=dev)
        self._status = torch.zeros(N, dtype=torch.int32, device=dev)

    def __call__(self, stack, gs):
        env = self.env
        for name, t, shape in (('stack', stack, (env.N, 3, env.beam_mum)), ('gs', gs, (env.N, 4))):
            if tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous() or t.device != env.device:
                raise ValueError(f'{name} must be a contiguous {shape} float32 tensor on {env.device}')
        _lib.check(env.lib.rlca_dwa_action(C.byref(env.cfg), C.byref(self._p), _ptr(self.directions), _ptr(stack),
                                           _ptr(gs), _ptr(self.action), _ptr(self._status), env._stream()))
        return self.action

    def status(self):
        """(N) int32 of the last call: 0 = the best admissible candidate, 1 = none was admissible, (0, 0) commanded."""
        return self._status

    def settings(self):
        return asdict(self.params)


def dwa_host(cfg, stack, gs, params=None, debug=False):
    """rlca_dwa_action_host on numpy arrays (stack (N, 3, beams), gs (N, 4) float32): (action (N, 2), status (N)), and
    with debug also every candidate's clearance and score, (N, v_samples w_samples) each, candidate iv w_samples + iw."""
    lib = _lib.load()
    params = DwaParams() if params is None else params
    n = int(cfg.robots_per_world) * int(cfg.num_worlds)
    s = np.ascontiguousarray(stack, np.float32)
    g = np.ascontiguousarray(gs, np.float32)
    if s.shape != (n, 3, int(cfg.beams)) or g.shape != (n, 4):
        raise ValueError(f'stack must be ({n}, 3, {int(cfg.beams)}) and gs ({n}, 4)')
    cs = beam_directions(cfg)
    act = np.zeros((n, 2), np.float32)
    status = np.zeros(n, np.int32)
    nc = params.v_samples * params.w_samples
    clear = np.zeros((n, nc), np.float32) if debug else None
    score = np.zeros((n, nc), np.float32) if debug else None
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    _lib.check(lib.rlca_dwa_action_host(C.byref(cfg), C.byref(params.struct()), vp(cs), vp(s), vp(g), vp(act),
                                        vp(status), vp(clear), vp(score)))
    return (act, status, clear, score) if debug else (act, status)


# ------------------------------------------------------------------------------------------------ command line
DWA_FLAGS = ('--dwa-radius', '--dwa-horizon', '--dwa-heading-time', '--dwa-samples', '--dwa-accel', '--dwa-brake',
             '--dwa-weights')
# the ORCA baselines' flags (orca.add_arguments), which do not apply to the dynamic window
ORCA_DESTS = ('orca_radius', 'orca_horizon', 'orca_neighbour_dist', 'orca_gain', 'nh_error', 'nh_heading_time',
              'orca_map', 'orca_obstacle_horizon')


def add_arguments(ap):
    """The --dwa-* flags of evaluate.py on an argparse parser (--baseline dwa is the driver's own)."""
    d = DwaParams()
    ap.add_argument('--dwa-radius', type=float, default=None, metavar='R',
                    help='dwa: robot disc radius, m (default %g)' % d.radius)
    ap.add_argument('--dwa-horizon', type=float, default=None, metavar='T',
                    help='dwa: arc simulated per candidate, s (default %g)' % d.horizon)
    ap.add_argument('--dwa-heading-time', type=float, default=None, metavar='T',
                    help='dwa: the goal bearing is scored from the pose after T s (default %g)' % d.heading_time)
    ap.add_argument('--dwa-samples', default=None, metavar='V,W',
                    help='dwa: candidate grid (default %d,%d)' % (d.v_samples, d.w_samples))
    ap.add_argument('--dwa-accel', default=None, metavar='A[,B]',
                    help='dwa: window half-widths A dt and B dt (B defaults to A); 0 = the whole action box (default)')
    ap.add_argument('--dwa-brake', type=float, default=None, metavar='B',
                    help='dwa: braking deceleration of the admissibility test, m/s^2 (default %g)' % d.brake)
    ap.add_argument('--dwa-weights', default=None, metavar='H,C,S',
                    help='dwa: heading, clearance and speed weights (default %g,%g,%g)'
                         % (d.heading_weight, d.clearance_weight, d.speed_weight))


def _numbers(text, n_min, n_max, kind=float):
    parts = text.split(',')
    if not n_min <= len(parts) <= n_max:
        raise ValueError('expected %s comma-separated values' % (n_min if n_min == n_max else '%d to %d' % (n_min, n_max)))
    return [kind(p) for p in parts]


def check_arguments(ap, args):
    """ap.error for a --dwa-* flag without --baseline dwa, and for an --orca-* / --nh-* flag set to anything but its
    default with it."""
    if args.baseline != 'dwa':
        given = [f for f in DWA_FLAGS if getattr(args, f[2:].replace('-', '_')) is not None]
        if given:
            ap.error('%s applies to --baseline dwa only' % given[0])
        return
    for dest in ORCA_DESTS:
        if getattr(args, dest) != ap.get_default(dest):
            ap.error('--%s applies to --baseline orca / nh-orca only, not dwa' % dest.replace('_', '-'))


def from_arguments(ap, args):
    """DwaParams of the --dwa-* flags, or None without --baseline dwa; ap.error for a bad value."""
    if args.baseline != 'dwa':
        return None
    kw = {}
    for flag in ('radius', 'horizon', 'heading_time', 'brake'):
        if getattr(args, 'dwa_' + flag) is not None:
            kw[flag] = getattr(args, 'dwa_' + flag)
    try:
        if args.dwa_samples is not None:
            kw['v_samples'], kw['w_samples'] = _numbers(args.dwa_samples, 2, 2, int)
        if args.dwa_accel is not None:
            a = _numbers(args.dwa_accel, 1, 2)
            kw['accel'], kw['angular_accel'] = a[0], a[-1]
        if args.dwa_weights is not None:
            kw['heading_weight'], kw['clearance_weight'], kw['speed_weight'] = _numbers(args.dwa_weights, 3, 3)
        return DwaParams(**kw)
    except ValueError as e:
        ap.error('--baseline dwa: %s' % e)
