"""Baseline controllers, one action per agent per tick:

- ORCA-DD (DESIGN.md §9d): reciprocal velocity obstacles over the robots of each world (van den Berg et al. 2011)
  followed by a differential-drive heading tracker;
- NH-ORCA (DESIGN.md §9e), the paper's baseline: ORCA restricted to the velocities a differential-drive robot tracks
  within an error E, radii grown by E, and the arc that tracks the chosen velocity (Alonso-Mora et al. 2010).

Both see only the other robots unless `obstacles=True`: then the static map's boundary adds RVO2's obstacle half-planes
with horizon `obstacle_time_horizon` (DESIGN.md §9f).

    ctrl = OrcaController(env)             # defaults: DEFAULTS below; NhOrcaController(env): NH_DEFAULTS
    action = ctrl()                        # (N, 2) raw (v, w) for env.control_vel, on the env's stream
    ctrl.velocities(), ctrl.status()       # ORCA velocities (N, 2) and LP status (N) of the last call
    OrcaController(env, obstacles=True)    # map-aware; status bits as STATUS_* below

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
# tau_o, s: with v_max = 1 m/s and r_o = 0.35 m the obstacle range is 1.35 m; a starting value, not a tuned one (§9f)
OBSTACLE_TIME_HORIZON = 1.0
MAP_MAX_LINES = 64              # RLCA_ORCA_MAP_MAX_LINES
# status bits of the map-aware controllers (bit 0 alone for the map-blind ones)
STATUS_FALLBACK, STATUS_OBSTACLE_FALLBACK, STATUS_DROPPED = 1, 2, 4


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def obstacle_range(cfg, obstacle_radius, obstacle_time_horizon):
    """tau_o * v_max + r_o in float32, as the library computes it."""
    f = np.float32
    return float(f(obstacle_time_horizon) * f(cfg.v_max) + f(obstacle_radius))


class ObstacleSet:
    """The static map's boundary segments and lookup bins (rlca_orca_obstacles_create): `cells` (H, W) uint8, 0 = free,
    with the resolution and origin of `cfg`; answers queries up to `max_range` m.  No device is needed to build it."""

    def __init__(self, cfg, cells, max_range):
        self.lib = _lib.load()
        c = np.ascontiguousarray(cells, np.uint8)
        if c.ndim != 2:
            raise ValueError('cells must be (H, W)')
        self.max_range = float(max_range)
        self.handle = C.c_void_p()
        _lib.check(self.lib.rlca_orca_obstacles_create(C.byref(cfg), c.ctypes.data_as(C.c_void_p), c.shape[1],
                                                       c.shape[0], self.max_range, C.byref(self.handle)))

    def segments(self):
        """(points (S, 4) float32 x0, y0, x1, y1; links (S, 3) int32 previous, next, convex start vertex; longest
        bin list)."""
        n, ml = C.c_int32(0), C.c_int32(0)
        _lib.check(self.lib.rlca_orca_obstacles_segments(self.handle, C.byref(n), C.byref(ml), None, None))
        pts = np.zeros((n.value, 4), np.float32)
        links = np.zeros((n.value, 3), np.int32)
        _lib.check(self.lib.rlca_orca_obstacles_segments(self.handle, C.byref(n), C.byref(ml),
                                                         pts.ctypes.data_as(C.c_void_p),
                                                         links.ctypes.data_as(C.c_void_p)))
        return pts, links, ml.value

    def lines(self, cfg, pose, goal, meta, agent, obstacle_radius, obstacle_time_horizon=OBSTACLE_TIME_HORIZON):
        """The obstacle lines of one agent ((k, 4) float32 point, unit direction; allowed side on the left) and
        whether lines were dropped at MAP_MAX_LINES."""
        p, g, m = (np.ascontiguousarray(a, t) for a, t in ((pose, np.float32), (goal, np.float32), (meta, np.int32)))
        out = np.zeros((MAP_MAX_LINES, 4), np.float32)
        n, d = C.c_int32(0), C.c_int32(0)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(self.lib.rlca_orca_obstacle_lines_host(C.byref(cfg), self.handle, vp(p), vp(g), vp(m), int(agent),
                                                          float(obstacle_radius), float(obstacle_time_horizon),
                                                          C.byref(n), C.byref(d), vp(out)))
        return out[:n.value].copy(), bool(d.value)

    def close(self):
        if self.handle:
            _lib.check(self.lib.rlca_orca_obstacles_destroy(self.handle))
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Controller:
    """Actions for every agent of a StageWorld from its current state.  Buffers are allocated once; each call
    overwrites them, so the returned action is valid until the next call.  With `obstacles` the map-aware entry runs
    on an ObstacleSet built from env.sc.map for this controller's obstacle range."""

    _entry = None

    def __init__(self, env, params, obstacles=False, obstacle_radius=None, obstacle_time_horizon=None):
        self.env = env
        self.params = tuple(float(p) for p in params)
        N, dev = env.N, env.device
        self.action = torch.zeros(N, 2, device=dev)
        self._velocity = torch.zeros(N, 2, device=dev)
        self._status = torch.zeros(N, dtype=torch.int32, device=dev)
        self.obstacles = None
        if obstacles:
            self.obstacle_time_horizon = float(obstacle_time_horizon)
            with torch.cuda.device(dev):
                self.obstacles = ObstacleSet(env.cfg, env.sc.map.cells,
                                             obstacle_range(env.cfg, obstacle_radius, obstacle_time_horizon))

    def __call__(self):
        env = self.env
        st = env._state_struct(env._cur)
        if self.obstacles is None:
            _lib.check(getattr(env.lib, self._entry)(C.byref(env.cfg), C.byref(st), *self.params, _ptr(self.action),
                                                     _ptr(self._velocity), _ptr(self._status), env._stream()))
        else:
            _lib.check(getattr(env.lib, self._entry + '_map')(C.byref(env.cfg), C.byref(st), self.obstacles.handle,
                                                              *self.params, self.obstacle_time_horizon,
                                                              _ptr(self.action), _ptr(self._velocity),
                                                              _ptr(self._status), env._stream()))
        return self.action

    def velocities(self):
        """(N, 2) ORCA velocities (world frame) of the last call."""
        return self._velocity

    def status(self):
        """(N) int32 of the last call: 0 = the LP was feasible, 1 = least-penetration fallback; map-aware, the bits
        STATUS_FALLBACK, STATUS_OBSTACLE_FALLBACK and STATUS_DROPPED."""
        return self._status


class OrcaController(_Controller):
    """ORCA-DD (rlca_orca_action)."""

    _entry = 'rlca_orca_action'

    def __init__(self, env, radius=DEFAULTS['radius'], neighbour_dist=DEFAULTS['neighbour_dist'],
                 time_horizon=DEFAULTS['time_horizon'], heading_gain=DEFAULTS['heading_gain'], obstacles=False,
                 obstacle_time_horizon=OBSTACLE_TIME_HORIZON):
        super().__init__(env, (radius, neighbour_dist, time_horizon, heading_gain), obstacles, radius,
                         obstacle_time_horizon)


class NhOrcaController(_Controller):
    """NH-ORCA (rlca_nh_orca_action)."""

    _entry = 'rlca_nh_orca_action'

    def __init__(self, env, radius=NH_DEFAULTS['radius'], neighbour_dist=NH_DEFAULTS['neighbour_dist'],
                 time_horizon=NH_DEFAULTS['time_horizon'], tracking_error=NH_DEFAULTS['tracking_error'],
                 heading_time=NH_DEFAULTS['heading_time'], obstacles=False,
                 obstacle_time_horizon=OBSTACLE_TIME_HORIZON):
        super().__init__(env, (radius, neighbour_dist, time_horizon, tracking_error, heading_time), obstacles,
                         np.float32(radius) + np.float32(tracking_error), obstacle_time_horizon)


def _host(entry, cfg, pose, goal, meta, params, obstacles=None, obstacle_time_horizon=OBSTACLE_TIME_HORIZON):
    """obstacles: None / False (map-blind) or an ObstacleSet (the _map entry)."""
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
    if obstacles:
        _lib.check(getattr(lib, entry.replace('_host', '_map_host'))(
            C.byref(cfg), obstacles.handle, vp(p), vp(g), vp(m), *(float(x) for x in params),
            float(obstacle_time_horizon), vp(act), vp(vel), vp(status)))
    else:
        _lib.check(getattr(lib, entry)(C.byref(cfg), vp(p), vp(g), vp(m), *(float(x) for x in params), vp(act),
                                       vp(vel), vp(status)))
    return act, vel, status


def orca_host(cfg, pose, goal, meta, radius=DEFAULTS['radius'], neighbour_dist=DEFAULTS['neighbour_dist'],
              time_horizon=DEFAULTS['time_horizon'], heading_gain=DEFAULTS['heading_gain'], obstacles=None,
              obstacle_time_horizon=OBSTACLE_TIME_HORIZON):
    """rlca_orca_action_host on numpy state arrays (pose, goal (N, 4) float32, meta (N, 4) int32); with an
    ObstacleSet `obstacles`, rlca_orca_action_map_host.  Returns (action (N, 2), velocity (N, 2), status (N))."""
    return _host('rlca_orca_action_host', cfg, pose, goal, meta, (radius, neighbour_dist, time_horizon, heading_gain),
                 obstacles, obstacle_time_horizon)


def nh_orca_host(cfg, pose, goal, meta, radius=NH_DEFAULTS['radius'], neighbour_dist=NH_DEFAULTS['neighbour_dist'],
                 time_horizon=NH_DEFAULTS['time_horizon'], tracking_error=NH_DEFAULTS['tracking_error'],
                 heading_time=NH_DEFAULTS['heading_time'], obstacles=None,
                 obstacle_time_horizon=OBSTACLE_TIME_HORIZON):
    """rlca_nh_orca_action_host (with an ObstacleSet: rlca_nh_orca_action_map_host) on numpy state arrays, as
    orca_host."""
    return _host('rlca_nh_orca_action_host', cfg, pose, goal, meta,
                 (radius, neighbour_dist, time_horizon, tracking_error, heading_time), obstacles, obstacle_time_horizon)


def nh_orca_polygon(cfg, tracking_error=NH_DEFAULTS['tracking_error'], heading_time=NH_DEFAULTS['heading_time']):
    """NH-ORCA's velocity polygon P in the robot frame (x along the heading): (k, 2) float32 vertices,
    counter-clockwise, for the bounds of `cfg`."""
    lib = _lib.load()
    verts = np.zeros((NH_ORCA_VERTS, 2), np.float32)
    nv = C.c_int32(0)
    _lib.check(lib.rlca_nh_orca_polygon_host(C.byref(cfg), float(tracking_error), float(heading_time), C.byref(nv),
                                             verts.ctypes.data_as(C.c_void_p)))
    return verts[:nv.value].copy()
