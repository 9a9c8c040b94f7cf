"""A global planner on the device (DESIGN.md §9w): the geodesic field of each robot's goal, a line-of-sight waypoint
as the policy's local goal where the goal is out of sight, and the geodesic length of every episode.

    planner = Planner(env, steer=True)        # the map's planning graph, uploaded once
    gs = planner.update(flags)                # after each tick (None at a run's start): the gs the policy reads

The graph (build_plan_tables, host, numpy and scipy, once per map): the traversable cells are the arena generator's
placeable cells (arenas.placeable_mask: a footprint centred anywhere in the cell, at any heading, covers free cells
only), moves go to the 8 neighbours at cost 70 (orthogonal) or 99 (diagonal, only where both orthogonal neighbours
are traversable), and every 4-connected component keeps its bounding rectangle.  A goal's field spans its component's
rectangle in one CTA's shared memory, so a map whose largest rectangle exceeds RLCA_PLAN_MAX_CELLS cells is refused.

Kernels: csrc/rlca_plan.cu (rlca_plan_fields, rlca_plan_waypoints, rlca_plan_track, rlca_plan_reduce).  The host
twins below run the same code on the CPU and equal the kernels bit for bit.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch
from scipy import ndimage

from . import _lib
from .arenas import placeable_mask

MAX_CELLS = 58112           # RLCA_PLAN_MAX_CELLS: 227 KB of shared memory per CTA on sm_90a at 4 bytes per cell
CHAIN_STEPS = 64            # the descent chain of rlca_plan_waypoints: two cells per lane of a warp
PARTIALS = _lib.PLAN_PARTIALS
NPARTIALS = len(PARTIALS)
STATUS_NAMES = ('goal_visible', 'waypoint', 'no_plan')
INF = 0xFFFFFFFF


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _vp(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


@dataclass(frozen=True)
class PlannerTables:
    """The planning graph of a map, as rlca_plan_tables holds it."""
    label: np.ndarray          # (grid_h, grid_w) int32: component of each traversable cell, -1 elsewhere
    rects: np.ndarray          # (K, 4) int32: cx0, cy0, cx1, cy1 (inclusive) of each component
    name: str = ''

    @property
    def count(self):
        return int(len(self.rects))

    @property
    def max_area(self):
        r = self.rects.astype(np.int64)
        return int(((r[:, 2] - r[:, 0] + 1) * (r[:, 3] - r[:, 1] + 1)).max())

    def struct(self, label_ptr=None, rects_ptr=None):
        """rlca_plan_tables of these tables: host pointers, or the given device pointers."""
        return _lib.PlanTables(self.count, self.max_area,
                               self.label.ctypes.data if label_ptr is None else label_ptr,
                               self.rects.ctypes.data if rects_ptr is None else rects_ptr)


def build_plan_tables(world_map):
    """PlannerTables of a WorldMap.  ValueError, naming the map and the limit, when the map has no traversable cell or
    a component's bounding rectangle holds more than MAX_CELLS cells."""
    name = world_map.name or 'the map'
    trav = placeable_mask(world_map.cells, world_map.resolution)
    lab, k = ndimage.label(trav)                     # 4-connected
    if k == 0:
        raise ValueError(f'planner: {name} has no traversable cell')
    rects = np.array([(s[1].start, s[0].start, s[1].stop - 1, s[0].stop - 1) for s in ndimage.find_objects(lab)],
                     np.int32)
    area = (rects[:, 2].astype(np.int64) - rects[:, 0] + 1) * (rects[:, 3].astype(np.int64) - rects[:, 1] + 1)
    big = int(np.argmax(area))
    if area[big] > MAX_CELLS:
        w, h = int(rects[big, 2] - rects[big, 0] + 1), int(rects[big, 3] - rects[big, 1] + 1)
        raise ValueError(f'planner: {name} is too big to plan on: a component spans a {w} x {h} = {int(area[big])}-cell '
                         f'rectangle, over the {MAX_CELLS}-cell limit of one field (227 KB of shared memory per CTA at '
                         f'4 bytes per cell)')
    return PlannerTables(np.ascontiguousarray(lab.astype(np.int32) - 1), rects, name)


def check_tables(cfg, tables):
    """rlca_plan_tables_check on the host tables."""
    _lib.check(_lib.load().rlca_plan_tables_check(C.byref(cfg), C.byref(tables.struct())))


class Planner:
    """The global planner of one StageWorld.  `update(flags)` after every tick (None at a run's start) re-plans the
    rows whose goal entry changed and, with `steer`, returns the gs the policy reads: env.gs where the goal is in sight
    or there is no plan, the waypoint's local goal elsewhere (one buffer reused by every call); without `steer` it
    returns env.gs.  `tables` are build_plan_tables(env.sc.map), built when None.  With a tracker attached (`attach`,
    as evaluate() does) it also keeps every episode's geodesic length, read at the tracker's episode boundaries: call
    update before the tracker's own track()."""

    def __init__(self, env, steer=True, tables=None):
        self.env, self.steer = env, bool(steer)
        self.tables = build_plan_tables(env.sc.map) if tables is None else tables
        check_tables(env.cfg, self.tables)
        N, dev = env.N, env.device
        self._label = torch.from_numpy(self.tables.label.reshape(-1)).to(dev)
        self._rects = torch.from_numpy(np.ascontiguousarray(self.tables.rects)).to(dev)
        self._t = self.tables.struct(self._label.data_ptr(), self._rects.data_ptr())
        self.entry = torch.full((N,), -1, dtype=torch.int32, device=dev)
        self.rect = torch.zeros(N, 4, dtype=torch.int32, device=dev)
        self.field = torch.empty(N, self.tables.max_area, dtype=torch.int32, device=dev)
        self.list = torch.zeros(N + 1, dtype=torch.int32, device=dev)
        self._status = torch.zeros(N, dtype=torch.uint8, device=dev)
        self.status_count = torch.zeros(N, 3, dtype=torch.int32, device=dev)
        self.gs = torch.zeros(N, 4, device=dev)
        self.tracker = self.length = self.records = None
        self._build_state()

    def _build_state(self):
        self._st = _lib.PlanState(_ptr(self.entry), _ptr(self.rect), _ptr(self.field), _ptr(self.list),
                                  _ptr(self._status), _ptr(self.status_count), _ptr(self.length), _ptr(self.records),
                                  self.tracker.episodes if self.tracker is not None else 0)

    def attach(self, tracker):
        """Keep the geodesic length of the episodes `tracker` (an EpisodeTracker of the same env) records, from the
        next update on; also zeroes the status counts."""
        if tracker.env is not self.env:
            raise ValueError('the tracker belongs to another env')
        self.tracker = tracker
        N, dev = self.env.N, self.env.device
        self.length = torch.full((N,), -1.0, device=dev)
        self.records = torch.full((N, tracker.episodes), -1.0, device=dev)
        self.status_count.zero_()
        self._build_state()

    def update(self, flags=None):
        """After a tick, with its env.flags (None at a run's start, before any tick): fields, waypoints (with steer)
        and the geodesic tracker (when attached), on the env's stream."""
        env = self.env
        cfg, stream = C.byref(env.cfg), env._stream()
        s_out = env._state_struct(env._cur)
        _lib.check(env.lib.rlca_plan_fields(cfg, C.byref(self._t), C.byref(self._st), C.byref(s_out), stream))
        if self.steer:
            _lib.check(env.lib.rlca_plan_waypoints(cfg, C.byref(self._t), C.byref(self._st), C.byref(s_out),
                                                   _ptr(env.gs), _ptr(self.gs), stream))
        if self.tracker is not None:
            if flags is not None and not env._ticked:
                raise RuntimeError('Planner.update(flags) needs a tick: call env.control_vel first')
            s_in = env._state_struct(1 - env._cur) if flags is not None else None
            _lib.check(env.lib.rlca_plan_track(cfg, C.byref(self._t), C.byref(self._st),
                                               C.byref(s_in) if s_in is not None else None, C.byref(s_out),
                                               _ptr(flags), C.byref(self.tracker._st), stream))
        return self.gs if self.steer else env.gs

    def status(self):
        """(N) uint8 of the last update with steer: 0 goal visible, 1 waypoint, 2 no plan."""
        return self._status

    def settings(self):
        t = self.tables
        return {'steer': self.steer, 'map': t.name, 'components': t.count, 'max_area': t.max_area,
                'chain_steps': CHAIN_STEPS}

    def status_shares(self, mask=None):
        """The share of robot-ticks with each status since attach (or construction), over the rows with mask 0 (all
        rows without a mask), and their number."""
        c = self.status_count.to(torch.int64)
        if mask is not None:
            c = c[torch.as_tensor(mask, device=c.device) == 0]
        tot = c.sum(0).cpu().numpy()
        n = int(tot.sum())
        out = {k: (int(v) / n if n else math.nan) for k, v in zip(STATUS_NAMES, tot)}
        out['robot_ticks'] = n
        return out

    def partials(self, world_begin=0, world_count=None, role_mask=None):
        """(world_count, NPARTIALS) float64 per-world geodesic partials of the attached tracker's records, or
        (world_count, 2, NPARTIALS) split by `role_mask` (N): row 0 over the agents with mask 0."""
        env = self.env
        if self.tracker is None:
            raise ValueError('the planner has no tracker attached')
        wc = env.num_worlds - world_begin if world_count is None else int(world_count)
        ev = C.byref(self.tracker._st)
        if role_mask is None:
            out = torch.empty(wc, NPARTIALS, dtype=torch.float64, device=env.device)
            _lib.check(env.lib.rlca_plan_reduce(C.byref(env.cfg), C.byref(self._st), ev, int(world_begin), wc,
                                                _ptr(out), env._stream()))
        else:
            m = torch.as_tensor(role_mask, device=env.device).to(torch.uint8).contiguous()
            if m.shape != (env.N,):
                raise ValueError(f'role_mask must have ({env.N},) entries')
            out = torch.empty(wc, 2, NPARTIALS, dtype=torch.float64, device=env.device)
            _lib.check(env.lib.rlca_plan_reduce_split(C.byref(env.cfg), C.byref(self._st), ev, _ptr(m),
                                                      int(world_begin), wc, _ptr(out), env._stream()))
        return out.cpu().numpy()


def geodesic_totals(partials):
    """Per-world geodesic partials (rows in global world order) summed left to right."""
    p = np.asarray(partials, np.float64).reshape(-1, NPARTIALS)
    tot = np.zeros(NPARTIALS, np.float64)
    for row in p:
        tot = tot + row
    return tot


def geodesic_metrics(tot):
    """Over the episodes that reached the goal with a path: their number, the mean geodesic length L and the mean and
    population std of the extra geodesic distance path - max(L - goal_radius, 0); and the recorded episodes whose start
    had no path."""
    t = dict(zip(PARTIALS, np.asarray(tot, np.float64).tolist()))
    n = t['reached']
    out = {'reached': int(n), 'no_path': int(t['no_path'])}
    if n:
        mean = t['sum_extra'] / n
        out['mean_length'] = t['sum_length'] / n
        out['extra_geodesic_distance'] = (mean, math.sqrt(max(t['sum_extra_sq'] / n - mean * mean, 0.0)))
    else:
        out['mean_length'] = math.nan
        out['extra_geodesic_distance'] = (math.nan, math.nan)
    return out


# ------------------------------------------------------------------------------------------------ host twins
class HostState:
    """Host buffers of rlca_plan_state for the host twins (the same layout as Planner's device buffers)."""

    def __init__(self, cfg, tables, episodes=1):
        N = int(cfg.robots_per_world) * int(cfg.num_worlds)
        self.entry = np.full(N, -1, np.int32)
        self.rect = np.zeros((N, 4), np.int32)
        self.field = np.zeros((N, tables.max_area), np.uint32)
        self.list = np.zeros(N + 1, np.int32)
        self.status = np.zeros(N, np.uint8)
        self.status_count = np.zeros((N, 3), np.int32)
        self.length = np.full(N, -1.0, np.float32)
        self.records = np.full((N, int(episodes)), -1.0, np.float32)
        self.episodes = int(episodes)

    def struct(self):
        return _lib.PlanState(*(a.ctypes.data for a in (self.entry, self.rect, self.field, self.list, self.status,
                                                         self.status_count, self.length, self.records)),
                              self.episodes)

    def replanned(self):
        """The rows the last fields_host call re-planned, ascending."""
        return self.list[1:1 + self.list[0]].copy()

    def row_field(self, a):
        """(h, w) uint32 field of row a over its rectangle."""
        x0, y0, x1, y1 = (int(v) for v in self.rect[a])
        w, h = x1 - x0 + 1, y1 - y0 + 1
        return self.field[a, :w * h].reshape(h, w)


def _f32(a, shape, name):
    a = np.ascontiguousarray(a, np.float32)
    if a.shape != shape:
        raise ValueError(f'{name} must have shape {shape}')
    return a


def fields_host(cfg, tables, state: HostState, goal):
    """rlca_plan_fields_host: re-plan the rows of `state` whose goal entry (from goal (N, 4)) changed."""
    N = len(state.entry)
    g = _f32(goal, (N, 4), 'goal')
    st = _lib.EnvState(None, g.ctypes.data, None, None)
    _lib.check(_lib.load().rlca_plan_fields_host(C.byref(cfg), C.byref(tables.struct()), C.byref(state.struct()),
                                                 C.byref(st)))
    return state


def waypoints_host(cfg, tables, state: HostState, pose, goal, gs_in):
    """rlca_plan_waypoints_host: gs_out (N, 4) float32; state.status and state.status_count updated."""
    N = len(state.entry)
    p, g, s = _f32(pose, (N, 4), 'pose'), _f32(goal, (N, 4), 'goal'), _f32(gs_in, (N, 4), 'gs_in')
    out = np.zeros_like(s)
    st = _lib.EnvState(p.ctypes.data, g.ctypes.data, None, None)
    _lib.check(_lib.load().rlca_plan_waypoints_host(C.byref(cfg), C.byref(tables.struct()), C.byref(state.struct()),
                                                    C.byref(st), _vp(s), _vp(out)))
    return out


def track_host(cfg, tables, state: HostState, acc_out, meta_in=None, flags=None, closed=None, count=None):
    """rlca_plan_track_host: with flags None every row's length from its init pose (acc_out[:, 2:4]); else the
    records of the tracked episodes that ended and the lengths of the re-spawned rows.  state updated in place."""
    N = len(state.entry)
    acc = _f32(acc_out, (N, 4), 'acc_out')
    s_out = _lib.EnvState(None, None, acc.ctypes.data, None)
    if flags is None:
        _lib.check(_lib.load().rlca_plan_track_host(C.byref(cfg), C.byref(tables.struct()), C.byref(state.struct()),
                                                    None, C.byref(s_out), None, None, None, state.episodes))
        return state
    mi = np.ascontiguousarray(meta_in, np.int32)
    fl = np.ascontiguousarray(flags, np.uint8)
    cl, cn = np.ascontiguousarray(closed, np.int32), np.ascontiguousarray(count, np.int32)
    if mi.shape != (N, 4) or fl.shape != (N, 4) or cl.shape != (N,) or cn.shape != (N,):
        raise ValueError('meta_in and flags must be (N, 4), closed and count (N)')
    s_in = _lib.EnvState(None, None, None, mi.ctypes.data)
    _lib.check(_lib.load().rlca_plan_track_host(C.byref(cfg), C.byref(tables.struct()), C.byref(state.struct()),
                                                C.byref(s_in), C.byref(s_out), _vp(fl), _vp(cl), _vp(cn),
                                                state.episodes))
    return state


def reduce_host(cfg, geo_records, eval_records, count, role_mask=None, world_begin=0, world_count=None):
    """rlca_plan_reduce_host: (world_count, NPARTIALS), or (world_count, 2, NPARTIALS) with a mask."""
    geo = np.ascontiguousarray(geo_records, np.float32)
    erec = np.ascontiguousarray(eval_records, np.float32)
    cnt = np.ascontiguousarray(count, np.int32)
    msk = None if role_mask is None else np.ascontiguousarray(role_mask, np.uint8)
    if erec.shape != geo.shape + (4,) or cnt.shape != geo.shape[:1] or (msk is not None and msk.shape != cnt.shape):
        raise ValueError('geo_records (N, E), eval_records (N, E, 4), count and role_mask (N) must match')
    wc = cfg.num_worlds - world_begin if world_count is None else int(world_count)
    out = np.zeros((wc, NPARTIALS) if msk is None else (wc, 2, NPARTIALS), np.float64)
    _lib.check(_lib.load().rlca_plan_reduce_host(C.byref(cfg), _vp(geo), _vp(erec), _vp(cnt), _vp(msk), geo.shape[1],
                                                 int(world_begin), wc, _vp(out)))
    return out


# ------------------------------------------------------------------------------------------------ command line
def add_arguments(ap):
    """--planner and --geodesic of evaluate.py on an argparse parser."""
    ap.add_argument('--planner', action='store_true',
                    help='steer the policy (or --baseline dwa) by a global planner on the device: where the goal is out '
                         'of sight its local goal is a waypoint on the geodesic path; also reports the geodesic '
                         'metrics (DESIGN.md §9w)')
    ap.add_argument('--geodesic', action='store_true',
                    help='report the geodesic length of every episode and the extra geodesic distance, without '
                         'steering (any controller; DESIGN.md §9w)')


def check_arguments(ap, args, localization=False):
    """ap.error for --planner together with --baseline orca / nh-orca, --hybrid or localization error (`localization`:
    a localization flag was given), and for --planner with --geodesic."""
    if not args.planner:
        return
    if args.geodesic:
        ap.error('--planner already reports the geodesic metrics; give one of --planner and --geodesic')
    if getattr(args, 'baseline', None) in ('orca', 'nh-orca'):
        ap.error('--planner steers what a policy reads; the ORCA baselines read the true goal through their own '
                 'kernels (use --geodesic)')
    if getattr(args, 'hybrid', False):
        ap.error('--planner steers what a policy reads; the hybrid driver reads the true goal (use --geodesic)')
    if localization:
        ap.error('--planner plans from the true pose; localization error needs a planner on the believed pose')


def from_arguments(args):
    """steer (True for --planner, False for --geodesic) or None."""
    return True if args.planner else False if args.geodesic else None
