"""Baseline controllers, one action per agent per tick:

- ORCA-DD (DESIGN.md §9d): reciprocal velocity obstacles over the robots of each world (van den Berg et al. 2011)
  followed by a differential-drive heading tracker;
- NH-ORCA (DESIGN.md §9e), the paper's baseline: ORCA restricted to the velocities a differential-drive robot tracks
  within an error E, radii grown by E, and the arc that tracks the chosen velocity (Alonso-Mora et al. 2010).

    ctrl = OrcaController(env)             # defaults: DEFAULTS below; NhOrcaController(env): NH_DEFAULTS
    action = ctrl()                        # (N, 2) raw (v, w) for env.control_vel, on the env's stream
    ctrl.velocities(), ctrl.status()       # ORCA velocities (N, 2) and LP status (N) of the last call

The controllers are csrc/rlca_orca.cu; `orca_host` / `nh_orca_host` run the same code on the CPU from numpy arrays.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

# radius: the footprint's circumscribed radius sqrt(0.22^2 + 0.19^2) = 0.2907 m plus a margin; neighbour_dist: the
# lidar range; fixed on the K = 4, r = 4 m circle swap (DESIGN.md §9d)
DEFAULTS = dict(radius=0.35, neighbour_dist=6.0, time_horizon=2.0, heading_gain=2.0)
# radius: the circumscribed 0.2907 m rounded up, so that radius + tracking_error is ORCA-DD's 0.35 m; starting values,
# not tuned ones (DESIGN.md §9e)
NH_DEFAULTS = dict(radius=0.30, neighbour_dist=6.0, time_horizon=2.0, tracking_error=0.05, heading_time=0.4)
NH_ORCA_VERTS = 32


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class _Controller:
    """Actions for every agent of a StageWorld from its current state.  Buffers are allocated once; each call
    overwrites them, so the returned action is valid until the next call."""

    _entry = None

    def __init__(self, env, params):
        self.env = env
        self.params = tuple(float(p) for p in params)
        N, dev = env.N, env.device
        self.action = torch.zeros(N, 2, device=dev)
        self._velocity = torch.zeros(N, 2, device=dev)
        self._status = torch.zeros(N, dtype=torch.int32, device=dev)

    def __call__(self):
        env = self.env
        st = env._state_struct(env._cur)
        _lib.check(getattr(env.lib, self._entry)(C.byref(env.cfg), C.byref(st), *self.params, _ptr(self.action),
                                                 _ptr(self._velocity), _ptr(self._status), env._stream()))
        return self.action

    def velocities(self):
        """(N, 2) ORCA velocities (world frame) of the last call."""
        return self._velocity

    def status(self):
        """(N) int32 of the last call: 0 = the LP was feasible, 1 = least-penetration fallback."""
        return self._status


class OrcaController(_Controller):
    """ORCA-DD (rlca_orca_action)."""

    _entry = 'rlca_orca_action'

    def __init__(self, env, radius=DEFAULTS['radius'], neighbour_dist=DEFAULTS['neighbour_dist'],
                 time_horizon=DEFAULTS['time_horizon'], heading_gain=DEFAULTS['heading_gain']):
        super().__init__(env, (radius, neighbour_dist, time_horizon, heading_gain))


class NhOrcaController(_Controller):
    """NH-ORCA (rlca_nh_orca_action)."""

    _entry = 'rlca_nh_orca_action'

    def __init__(self, env, radius=NH_DEFAULTS['radius'], neighbour_dist=NH_DEFAULTS['neighbour_dist'],
                 time_horizon=NH_DEFAULTS['time_horizon'], tracking_error=NH_DEFAULTS['tracking_error'],
                 heading_time=NH_DEFAULTS['heading_time']):
        super().__init__(env, (radius, neighbour_dist, time_horizon, tracking_error, heading_time))


def _host(entry, cfg, pose, goal, meta, params):
    lib = _lib.load()
    p = np.ascontiguousarray(pose, np.float32)
    g = np.ascontiguousarray(goal, np.float32)
    m = np.ascontiguousarray(meta, np.int32)
    n = cfg.robots_per_world * cfg.num_worlds
    if p.shape != (n, 4) or g.shape != (n, 4) or m.shape != (n, 4):
        raise ValueError(f'pose, goal and meta must be ({n}, 4)')
    act = np.zeros((n, 2), np.float32)
    vel = np.zeros((n, 2), np.float32)
    status = np.zeros(n, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(getattr(lib, entry)(C.byref(cfg), vp(p), vp(g), vp(m), *(float(x) for x in params), vp(act), vp(vel),
                                   vp(status)))
    return act, vel, status


def orca_host(cfg, pose, goal, meta, radius=DEFAULTS['radius'], neighbour_dist=DEFAULTS['neighbour_dist'],
              time_horizon=DEFAULTS['time_horizon'], heading_gain=DEFAULTS['heading_gain']):
    """rlca_orca_action_host on numpy state arrays (pose, goal (N, 4) float32, meta (N, 4) int32).
    Returns (action (N, 2), velocity (N, 2), status (N))."""
    return _host('rlca_orca_action_host', cfg, pose, goal, meta, (radius, neighbour_dist, time_horizon, heading_gain))


def nh_orca_host(cfg, pose, goal, meta, radius=NH_DEFAULTS['radius'], neighbour_dist=NH_DEFAULTS['neighbour_dist'],
                 time_horizon=NH_DEFAULTS['time_horizon'], tracking_error=NH_DEFAULTS['tracking_error'],
                 heading_time=NH_DEFAULTS['heading_time']):
    """rlca_nh_orca_action_host on numpy state arrays, as orca_host."""
    return _host('rlca_nh_orca_action_host', cfg, pose, goal, meta,
                 (radius, neighbour_dist, time_horizon, tracking_error, heading_time))


def nh_orca_polygon(cfg, tracking_error=NH_DEFAULTS['tracking_error'], heading_time=NH_DEFAULTS['heading_time']):
    """NH-ORCA's velocity polygon P in the robot frame (x along the heading): (k, 2) float32 vertices,
    counter-clockwise, for the bounds of `cfg`."""
    lib = _lib.load()
    verts = np.zeros((NH_ORCA_VERTS, 2), np.float32)
    nv = C.c_int32(0)
    _lib.check(lib.rlca_nh_orca_polygon_host(C.byref(cfg), float(tracking_error), float(heading_time), C.byref(nv),
                                             verts.ctypes.data_as(C.c_void_p)))
    return verts[:nv.value].copy()
