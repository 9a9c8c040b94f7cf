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

    nc = NonCooperative(env, mask)         # DESIGN.md §9h: masked robots drive straight to their goals
    nc.apply(action)                       # overwrites the masked rows of any controller's or policy's action

    hy = Hybrid(env)                       # DESIGN.md §9j: driver in free space, capped speed near obstacles
    hy.apply(action, stack, tracker)       # switches a policy's action by the nearest return of its newest scan
"""
from __future__ import annotations

import argparse
import ctypes as C
import math

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


def add_arguments(ap, map_default=False):
    """The controller flags of the command-line drivers (evaluate.py, sl_train.py) on an argparse parser; `--baseline`
    is the driver's own.  With map_default the map is on unless --no-orca-map."""
    ap.add_argument('--orca-radius', type=float, default=None,
                    help='robot radius, m (default %g for orca, %g for nh-orca)' % (DEFAULTS['radius'], NH_DEFAULTS['radius']))
    ap.add_argument('--orca-horizon', type=float, default=DEFAULTS['time_horizon'], help='time horizon tau, s')
    ap.add_argument('--orca-neighbour-dist', type=float, default=DEFAULTS['neighbour_dist'],
                    help='neighbours are the robots closer than this, m')
    ap.add_argument('--orca-gain', type=float, default=None,
                    help='ORCA-DD heading gain k_w, 1/s (default %g)' % DEFAULTS['heading_gain'])
    ap.add_argument('--nh-error', type=float, default=NH_DEFAULTS['tracking_error'], help='NH-ORCA tracking error E, m')
    ap.add_argument('--nh-heading-time', type=float, default=NH_DEFAULTS['heading_time'],
                    help='NH-ORCA heading time T, s')
    ap.add_argument('--orca-map', action=argparse.BooleanOptionalAction if map_default else 'store_true',
                    default=map_default,
                    help='the baseline also avoids the static map (obstacle half-planes from the occupancy grid)')
    ap.add_argument('--orca-obstacle-horizon', type=float, default=None,
                    help='obstacle time horizon tau_o, s, with --orca-map (default %g)' % OBSTACLE_TIME_HORIZON)


def check_arguments(ap, args):
    """ap.error() on controller flags that do not apply to args.baseline."""
    if args.baseline != 'orca' and args.orca_gain is not None:
        ap.error('--orca-gain applies to --baseline orca only')
    if not args.orca_map and args.orca_obstacle_horizon is not None:
        ap.error('--orca-obstacle-horizon applies with --orca-map only')


def from_arguments(env, args):
    """(controller, name) for args.baseline 'orca' or 'nh-orca' and the flags of add_arguments."""
    horizon = OBSTACLE_TIME_HORIZON if args.orca_obstacle_horizon is None else args.orca_obstacle_horizon
    if args.baseline == 'orca':
        gain = DEFAULTS['heading_gain'] if args.orca_gain is None else args.orca_gain
        radius = DEFAULTS['radius'] if args.orca_radius is None else args.orca_radius
        ctrl = OrcaController(env, radius=radius, neighbour_dist=args.orca_neighbour_dist,
                              time_horizon=args.orca_horizon, heading_gain=gain, obstacles=args.orca_map,
                              obstacle_time_horizon=horizon)
        return ctrl, 'orca-dd+map' if args.orca_map else 'orca-dd'
    if args.baseline == 'nh-orca':
        radius = NH_DEFAULTS['radius'] if args.orca_radius is None else args.orca_radius
        ctrl = NhOrcaController(env, radius=radius, neighbour_dist=args.orca_neighbour_dist,
                                time_horizon=args.orca_horizon, tracking_error=args.nh_error,
                                heading_time=args.nh_heading_time, obstacles=args.orca_map,
                                obstacle_time_horizon=horizon)
        return ctrl, 'nh-orca+map' if args.orca_map else 'nh-orca'
    raise ValueError('unknown baseline %r' % (args.baseline,))


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


class NonCooperative:
    """Non-cooperative robots (rlca_noncoop_action, DESIGN.md §9h): the agents with `mask` != 0 drive straight to their
    goals at `speed` (default cfg.v_max) with ORCA-DD's heading tracker (gain `heading_gain`), ignoring every other
    robot and the map.  `mask` (N) is held on the env's device as uint8."""

    def __init__(self, env, mask, speed=None, heading_gain=DEFAULTS['heading_gain']):
        self.env = env
        self.mask = torch.as_tensor(mask, device=env.device).to(torch.uint8).contiguous()
        if self.mask.shape != (env.N,):
            raise ValueError(f'mask must have ({env.N},) entries')
        self.speed = float(env.cfg.v_max) if speed is None else float(speed)
        self.heading_gain = float(heading_gain)

    def apply(self, action):
        """Overwrite the masked rows of `action` ((N, 2) float32, contiguous, on the env's device) in place, from the
        state the next tick reads, on the env's stream; returns `action`."""
        env = self.env
        if action.shape != (env.N, 2) or action.dtype != torch.float32 or not action.is_contiguous() or \
                action.device != self.mask.device:
            raise ValueError(f'action must be a contiguous ({env.N}, 2) float32 tensor on {self.mask.device}')
        st = env._state_struct(env._cur)
        _lib.check(env.lib.rlca_noncoop_action(C.byref(env.cfg), C.byref(st), _ptr(self.mask), self.speed,
                                               self.heading_gain, _ptr(action), env._stream()))
        return action


def noncoop_host(cfg, pose, goal, meta, mask, action, speed=None, heading_gain=DEFAULTS['heading_gain']):
    """rlca_noncoop_action_host on numpy arrays, as orca_host: returns a copy of `action` (N, 2) whose rows with
    mask != 0 are overwritten."""
    lib = _lib.load()
    p = np.ascontiguousarray(pose, np.float32)
    g = np.ascontiguousarray(goal, np.float32)
    m = np.ascontiguousarray(meta, np.int32)
    k = np.ascontiguousarray(mask, np.uint8)
    act = np.array(action, np.float32, order='C', copy=True)
    n = cfg.robots_per_world * cfg.num_worlds
    if p.shape != (n, 4) or g.shape != (n, 4) or m.shape != (n, 4) or k.shape != (n,) or act.shape != (n, 2):
        raise ValueError(f'pose, goal and meta must be ({n}, 4), mask ({n},) and action ({n}, 2)')
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_noncoop_action_host(C.byref(cfg), vp(p), vp(g), vp(m), vp(k),
                                            float(cfg.v_max) if speed is None else float(speed), float(heading_gain),
                                            vp(act)))
    return act


# starting values, not tuned ones (DESIGN.md §9j); heading_gain is the §9h driver's
HYBRID_DEFAULTS = dict(r_safe=2.0, r_risk=0.8, v_safe=0.5, heading_gain=2.0)
HYBRID_MODES = ('policy', 'driver', 'safe')      # mode 0, 1, 2


def check_hybrid(range_max, v_max, r_safe, r_risk, v_safe, heading_gain):
    """ValueError unless 0 <= r_risk <= r_safe <= range_max (all finite), 0 < v_safe <= v_max and heading_gain is
    finite and > 0: the rule rlca_hybrid_action applies, checked before any device work."""
    f = np.float32
    r_safe, r_risk, v_safe, gain, rm = (f(x) for x in (r_safe, r_risk, v_safe, heading_gain, range_max))
    if not (0.0 <= r_risk <= r_safe <= rm and math.isfinite(rm)):
        raise ValueError('hybrid radii need 0 <= r_risk <= r_safe <= range_max (%g), got r_risk %g, r_safe %g'
                         % (rm, r_risk, r_safe))
    if not 0.0 < v_safe <= f(v_max):
        raise ValueError('hybrid v_safe must be in (0, %g], got %g' % (f(v_max), v_safe))
    if not (gain > 0.0 and math.isfinite(gain)):
        raise ValueError('hybrid heading_gain must be finite and > 0, got %g' % gain)


class Hybrid:
    """The hybrid controller (rlca_hybrid_action, DESIGN.md §9j): per agent and tick, with d the nearest return of the
    newest scan in metres, the §9h driver at v_max when d > r_safe (mode 1), the policy's action with v capped at
    v_safe when d < r_risk (mode 2), the policy's action otherwise (mode 0).  Holds the per-agent mode counters (N, 3)
    int32 on the env's device; they count the ticks of the episodes an EpisodeTracker follows."""

    def __init__(self, env, r_safe=HYBRID_DEFAULTS['r_safe'], r_risk=HYBRID_DEFAULTS['r_risk'],
                 v_safe=HYBRID_DEFAULTS['v_safe'], heading_gain=HYBRID_DEFAULTS['heading_gain']):
        check_hybrid(env.cfg.range_max, env.cfg.v_max, r_safe, r_risk, v_safe, heading_gain)
        self.env = env
        self.params = _lib.HybridParams(r_safe, r_risk, v_safe, heading_gain)
        self.counts = torch.zeros(env.N, len(HYBRID_MODES), dtype=torch.int32, device=env.device)
        self.mode = torch.zeros(env.N, dtype=torch.uint8, device=env.device)

    def reset(self):
        """Zero the mode counters."""
        self.counts.zero_()

    def apply(self, action, stack, tracker=None):
        """Rewrite `action` ((N, 2) float32, contiguous) in place from `stack` ((N, 3, beams) float32, the scan FIFO
        the next tick reads) and the state the next tick reads, on the env's stream without synchronisation; with an
        EpisodeTracker, count each agent's mode when its `open` flag is set.  `self.mode` holds the modes; returns
        `action`."""
        env = self.env
        dev = self.counts.device
        if action.shape != (env.N, 2) or action.dtype != torch.float32 or not action.is_contiguous() or \
                action.device != dev:
            raise ValueError(f'action must be a contiguous ({env.N}, 2) float32 tensor on {dev}')
        if stack.shape != (env.N, 3, env.cfg.beams) or stack.dtype != torch.float32 or not stack.is_contiguous() or \
                stack.device != dev:
            raise ValueError(f'stack must be a contiguous ({env.N}, 3, {env.cfg.beams}) float32 tensor on {dev}')
        st = env._state_struct(env._cur)
        open_, counts = (tracker.open, self.counts) if tracker is not None else (None, None)
        _lib.check(env.lib.rlca_hybrid_action(C.byref(env.cfg), C.byref(self.params), C.byref(st), _ptr(stack),
                                              _ptr(open_), _ptr(action), _ptr(self.mode), _ptr(counts),
                                              env._stream()))
        return action

    def counts_per_world(self, mask=None):
        """(num_worlds, 3) int64 mode counts summed over each world's agents, over those with mask 0 when an agent
        mask (N) is given (exact integers, so shards give the same rows)."""
        c = self.counts.to(torch.int64)
        if mask is not None:
            keep = torch.as_tensor(mask, device=c.device) == 0
            if keep.shape != (self.env.N,):
                raise ValueError(f'mask must have ({self.env.N},) entries')
            c = c * keep[:, None]
        return c.view(self.env.num_worlds, -1, len(HYBRID_MODES)).sum(1).cpu().numpy()


def mode_shares(mode_counts):
    """{'policy', 'driver', 'safe': share of the counted agent-ticks (NaN when none), 'agent_ticks'} of (W, 3)
    counts."""
    tot = np.asarray(mode_counts, np.int64).reshape(-1, len(HYBRID_MODES)).sum(0)
    n = int(tot.sum())
    out = {name: (int(c) / n if n else math.nan) for name, c in zip(HYBRID_MODES, tot)}
    out['agent_ticks'] = n
    return out


def hybrid_host(cfg, stack, pose, goal, meta, action, open_=None, counts=None, r_safe=HYBRID_DEFAULTS['r_safe'],
                r_risk=HYBRID_DEFAULTS['r_risk'], v_safe=HYBRID_DEFAULTS['v_safe'],
                heading_gain=HYBRID_DEFAULTS['heading_gain']):
    """rlca_hybrid_action_host on numpy arrays (stack (N, 3, beams) float32, pose / goal / meta as orca_host): returns
    (action (N, 2), mode (N) uint8, counts (N, 3) int32), copies of `action` and `counts` (zeros when None) rewritten;
    counting happens only with `open_` (N)."""
    lib = _lib.load()
    n, beams = cfg.robots_per_world * cfg.num_worlds, cfg.beams
    s = np.ascontiguousarray(stack, np.float32)
    p = np.ascontiguousarray(pose, np.float32)
    g = np.ascontiguousarray(goal, np.float32)
    m = np.ascontiguousarray(meta, np.int32)
    act = np.array(action, np.float32, order='C', copy=True)
    cnt = np.zeros((n, len(HYBRID_MODES)), np.int32) if counts is None else np.array(counts, np.int32, order='C',
                                                                                       copy=True)
    opn = None if open_ is None else np.ascontiguousarray(open_, np.int32)
    if s.shape != (n, 3, beams) or p.shape != (n, 4) or g.shape != (n, 4) or m.shape != (n, 4) or \
            act.shape != (n, 2) or cnt.shape != (n, 3) or (opn is not None and opn.shape != (n,)):
        raise ValueError(f'stack must be ({n}, 3, {beams}), pose, goal and meta ({n}, 4), action ({n}, 2), '
                         f'open ({n},) and counts ({n}, 3)')
    mode = np.zeros(n, np.uint8)
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    prm = _lib.HybridParams(r_safe, r_risk, v_safe, heading_gain)
    _lib.check(lib.rlca_hybrid_action_host(C.byref(cfg), C.byref(prm), vp(s), vp(p), vp(g), vp(m), vp(opn), vp(act),
                                           vp(mode), vp(cnt if opn is not None else None)))
    return act, mode, cnt


def nh_orca_polygon(cfg, tracking_error=NH_DEFAULTS['tracking_error'], heading_time=NH_DEFAULTS['heading_time']):
    """NH-ORCA's velocity polygon P in the robot frame (x along the heading): (k, 2) float32 vertices,
    counter-clockwise, for the bounds of `cfg`."""
    lib = _lib.load()
    verts = np.zeros((NH_ORCA_VERTS, 2), np.float32)
    nv = C.c_int32(0)
    _lib.check(lib.rlca_nh_orca_polygon_host(C.byref(cfg), float(tracking_error), float(heading_time), C.byref(nv),
                                             verts.ctypes.data_as(C.c_void_p)))
    return verts[:nv.value].copy()
