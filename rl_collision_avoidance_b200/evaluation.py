"""Deterministic evaluation of a policy on any scenario, with the metrics of the paper the reference accompanies:
success rate, extra time, extra distance and average speed (DESIGN.md §9c).

    tracker = EpisodeTracker(env, episodes=E)     # device buffers; tracker.track() after every env tick
    out = evaluate(env, policy, episodes=E, max_ticks=T)
    out['partials']  (num_worlds, 14) float64 per-world partials (columns: _lib.EVAL_PARTIALS)
    out['totals']    the partials summed in world order;  out['metrics'] = metrics(out['totals'])

Records and partials come from librlca.so (csrc/rlca_eval.cu).  Totals of several shards (handles with world_offset,
or GPUs) are `totals(np.concatenate(partials in global world order))`, bit-identical to one handle's.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .dwa import DwaController
from .model.ppo import generate_action_no_sampling
from .orca import NhOrcaController, OrcaController, mode_shares
from .perturbation import Chain
from .planner import geodesic_metrics, geodesic_totals

COLUMNS = _lib.EVAL_PARTIALS
NPARTIALS = len(COLUMNS)
SAFETY_COLUMNS = _lib.SAFETY_PARTIALS
SAFETY_NPARTIALS = len(SAFETY_COLUMNS)
PROGRESS_COLUMNS = _lib.PROGRESS_PARTIALS
PROGRESS_NPARTIALS = len(PROGRESS_COLUMNS)
# DESIGN.md §9o: a third of stage 1's 150-tick budget; 10 cm of progress; 5 mm per tick (0.05 m/s at dt 0.1); 1 m
PROGRESS_DEFAULTS = {'window': 50, 'progress_dist': 0.1, 'still_dist': 0.005, 'block_dist': 1.0}
ACTION_BOUND = [[0, -1], [1, 1]]
# the reference's episode mechanics per scenario: stage 1 re-spawns a robot as soon as it is done
# (ppo_stage1.py:51-65), stage 2 re-spawns a group when all of it is done (ppo_stage2.py:49-106), circle runs one
# episode that the caller never resets (circle_test.py:36-84); so does the random scenario, one layout per world
AUTO_RESET = {'stage1': 1, 'stage2': 2, 'circle': 0, 'random': 0, 'arena': 0}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class EpisodeTracker:
    """Per-agent episode records of a StageWorld: call `track()` after each `env.control_vel`.  An agent's first
    `episodes` ended episodes are recorded (result code, ticks, path length, straight-line start -> goal distance);
    later ones are counted and dropped, and the episode running when evaluation stops is counted as unfinished."""

    def __init__(self, env, episodes):
        if int(episodes) < 1:
            raise ValueError('episodes must be >= 1')
        self.env, self.episodes = env, int(episodes)
        N, dev = env.N, env.device
        self.path = torch.zeros(N, dtype=torch.float64, device=dev)
        self.count = torch.zeros(N, dtype=torch.int32, device=dev)
        self.closed = torch.full((N,), -1, dtype=torch.int32, device=dev)
        self.open = torch.ones(N, dtype=torch.int32, device=dev)
        self.records = torch.zeros(N, self.episodes, 4, device=dev)
        self._st = _lib.EvalState(_ptr(self.path), _ptr(self.count), _ptr(self.closed), _ptr(self.open),
                                  _ptr(self.records), self.episodes)

    def reset(self):
        """Forget every record; the agents' running episodes are tracked from their current poses."""
        self.path.zero_()
        self.count.zero_()
        self.closed.fill_(-1)
        self.open.fill_(1)
        self.records.zero_()

    def track(self):
        """Records of the tick `env.control_vel` just ran (same stream, no synchronisation)."""
        env = self.env
        if not env._ticked:
            raise RuntimeError('EpisodeTracker.track() needs a tick: call env.control_vel first')
        s_in, s_out = env._state_struct(1 - env._cur), env._state_struct(env._cur)
        o = env._last_out
        io = env._io(action=env._keep[0], out=o)
        _lib.check(env.lib.rlca_eval_track(C.byref(env.cfg), C.byref(s_in), C.byref(s_out), C.byref(io),
                                           C.byref(self._st), env._stream()))

    def partials(self, world_begin=0, world_count=None):
        """(world_count, NPARTIALS) float64 per-world partials of worlds [world_begin, world_begin + world_count) of
        this handle, reduced on the device in a fixed order."""
        env = self.env
        wc = env.num_worlds - world_begin if world_count is None else int(world_count)
        out = torch.empty(wc, NPARTIALS, dtype=torch.float64, device=env.device)
        _lib.check(env.lib.rlca_eval_reduce(C.byref(env.cfg), C.byref(self._st), int(world_begin), wc, _ptr(out),
                                            env._stream()))
        return out.cpu().numpy()

    def partials_split(self, mask, world_begin=0, world_count=None):
        """(world_count, 2, NPARTIALS) per-world partials split by the agent mask (N): row 0 over the agents with mask
        0, row 1 over the others (rlca_eval_reduce_split)."""
        env = self.env
        wc = env.num_worlds - world_begin if world_count is None else int(world_count)
        m = torch.as_tensor(mask, device=env.device).to(torch.uint8).contiguous()
        if m.shape != (env.N,):
            raise ValueError(f'mask must have ({env.N},) entries')
        out = torch.empty(wc, 2, NPARTIALS, dtype=torch.float64, device=env.device)
        _lib.check(env.lib.rlca_eval_reduce_split(C.byref(env.cfg), C.byref(self._st), _ptr(m), int(world_begin), wc,
                                                  _ptr(out), env._stream()))
        return out.cpu().numpy()


def reduce_host(cfg, records, count, open_, world_begin=0, world_count=None):
    """rlca_eval_reduce on host arrays (the same code, run by the CPU): records (N, E, 4) float32, count and open (N)."""
    lib = _lib.load()
    rec = np.ascontiguousarray(records, np.float32)
    cnt = np.ascontiguousarray(count, np.int32)
    opn = np.ascontiguousarray(open_, np.int32)
    wc = cfg.num_worlds - world_begin if world_count is None else int(world_count)
    out = np.zeros((wc, NPARTIALS), np.float64)
    _lib.check(lib.rlca_eval_reduce_host(C.byref(cfg), rec.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p),
                                         opn.ctypes.data_as(C.c_void_p), rec.shape[1], int(world_begin), wc,
                                         out.ctypes.data_as(C.c_void_p)))
    return out


def reduce_split_host(cfg, records, count, open_, mask, world_begin=0, world_count=None):
    """rlca_eval_reduce_split on host arrays, as reduce_host, with the agent mask (N): (world_count, 2, NPARTIALS)."""
    lib = _lib.load()
    rec = np.ascontiguousarray(records, np.float32)
    cnt = np.ascontiguousarray(count, np.int32)
    opn = np.ascontiguousarray(open_, np.int32)
    msk = np.ascontiguousarray(mask, np.uint8)
    if msk.shape != cnt.shape:
        raise ValueError('mask must have one entry per agent')
    wc = cfg.num_worlds - world_begin if world_count is None else int(world_count)
    out = np.zeros((wc, 2, NPARTIALS), np.float64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_eval_reduce_split_host(C.byref(cfg), vp(rec), vp(cnt), vp(opn), vp(msk), rec.shape[1],
                                               int(world_begin), wc, vp(out)))
    return out


class SafetyTracker:
    """Per-episode safety records next to an EpisodeTracker's (DESIGN.md §9m): minimum separation between footprints
    and the robot it was to, minimum clearance (nearest scan return), near-miss ticks (separation below `near_dist`
    metres) and the cause of a crash.  Call `track()` after each `env.control_vel` and BEFORE `tracker.track()`: the
    episode a tick belongs to and the record slot are read from the tracker's state as its own call will see them."""

    def __init__(self, env, tracker, near_dist=0.1):
        near_dist = float(near_dist)
        if not (math.isfinite(near_dist) and near_dist >= 0.0):
            raise ValueError('near_dist must be finite and >= 0')
        self.env, self.tracker, self.near_dist = env, tracker, near_dist
        N, dev = env.N, env.device
        self.min_sep = torch.empty(N, device=dev)
        self.min_clear = torch.empty(N, device=dev)
        self.last_clear = torch.empty(N, device=dev)
        self.near = torch.empty(N, dtype=torch.int32, device=dev)
        self.partner = torch.empty(N, dtype=torch.int32, device=dev)
        self.records = torch.empty(N, tracker.episodes, 4, device=dev)
        self._params = _lib.SafetyParams(near_dist)
        self._st = _lib.SafetyState(_ptr(self.min_sep), _ptr(self.min_clear), _ptr(self.last_clear), _ptr(self.near),
                                    _ptr(self.partner), _ptr(self.records), tracker.episodes)
        self.reset()

    def reset(self):
        """Forget every record and the running episodes (with the tracker's own reset())."""
        for t in (self.min_sep, self.min_clear, self.last_clear):
            t.fill_(math.inf)
        self.near.zero_()
        self.partner.fill_(-1)
        self.records.zero_()

    def track(self):
        """Safety records of the tick `env.control_vel` just ran (same stream, no synchronisation)."""
        env = self.env
        if not env._ticked:
            raise RuntimeError('SafetyTracker.track() needs a tick: call env.control_vel first')
        s_in, s_out = env._state_struct(1 - env._cur), env._state_struct(env._cur)
        io = env._io(action=env._keep[0], out=env._last_out)
        _lib.check(env.lib.rlca_safety_track(C.byref(env.cfg), C.byref(self._params), C.byref(s_in), C.byref(s_out),
                                             C.byref(io), C.byref(self.tracker._st), C.byref(self._st),
                                             env._stream()))

    def partials(self, world_begin=0, world_count=None, role_mask=None):
        """(world_count, SAFETY_NPARTIALS) float64 per-world partials, or (world_count, 2, SAFETY_NPARTIALS) split by
        the agent mask `role_mask` (N): row 0 over the agents with mask 0, row 1 over the others, with the crashes
        charged to a masked robot counted in 'crash_into_masked'."""
        env = self.env
        wc = env.num_worlds - world_begin if world_count is None else int(world_count)
        m = None
        if role_mask is not None:
            m = torch.as_tensor(role_mask, device=env.device).to(torch.uint8).contiguous()
            if m.shape != (env.N,):
                raise ValueError(f'role_mask must have ({env.N},) entries')
        shape = (wc, SAFETY_NPARTIALS) if m is None else (wc, 2, SAFETY_NPARTIALS)
        out = torch.empty(shape, dtype=torch.float64, device=env.device)
        _lib.check(env.lib.rlca_safety_reduce(C.byref(env.cfg), C.byref(self._st), C.byref(self.tracker._st), _ptr(m),
                                              int(world_begin), wc, _ptr(out), env._stream()))
        return out.cpu().numpy()


def safety_contact(cfg):
    """The contact bound of a config in metres (float32, as the library computes it)."""
    out = C.c_float()
    _lib.check(_lib.load().rlca_safety_contact_host(C.byref(cfg), C.byref(out)))
    return np.float32(out.value)


def safety_separation_host(cfg, pose_a, pose_b):
    """Separation of the footprints at pose_a[i] and pose_b[i] ((n, 4) or (n, 3) x, y, theta), by the library's code."""
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    pad = lambda p: np.ascontiguousarray(np.concatenate(
        (np.asarray(p, np.float32)[:, :3], np.zeros((len(p), 1), np.float32)), 1))
    a, b = pad(pose_a), pad(pose_b)
    if a.shape != b.shape:
        raise ValueError('pose_a and pose_b must have the same number of rows')
    out = np.zeros(len(a), np.float32)
    _lib.check(_lib.load().rlca_safety_separation_host(C.byref(cfg), vp(a), vp(b), len(a), vp(out)))
    return out


def safety_track_host(cfg, near_dist, pose_in, meta_in, pose_out, flags, obs, closed, count, state):
    """rlca_safety_track on host arrays (the same code, run by the CPU).  `state` is a dict of min_sep, min_clear,
    last_clear (N) float32, near, partner (N) int32 and records (N, E, 4) float32, updated in place."""
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    for k, dt in (('min_sep', np.float32), ('min_clear', np.float32), ('last_clear', np.float32), ('near', np.int32),
                  ('partner', np.int32), ('records', np.float32)):
        if state[k].dtype != dt or not state[k].flags.c_contiguous:
            raise ValueError(f'state[{k!r}] must be a contiguous {np.dtype(dt).name} array')
    args = [f32(pose_in), i32(meta_in), f32(pose_out), np.ascontiguousarray(flags, np.uint8), f32(obs), i32(closed),
            i32(count)]
    _lib.check(_lib.load().rlca_safety_track_host(
        C.byref(cfg), C.byref(_lib.SafetyParams(float(near_dist))), *(vp(a) for a in args), state['records'].shape[1],
        *(vp(state[k]) for k in ('min_sep', 'min_clear', 'last_clear', 'near', 'partner', 'records'))))
    return state


def safety_reduce_host(cfg, safety_records, eval_records, count, role_mask=None, world_begin=0, world_count=None):
    """rlca_safety_reduce on host arrays: (world_count, SAFETY_NPARTIALS), or (world_count, 2, ...) with a mask."""
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    srec = np.ascontiguousarray(safety_records, np.float32)
    erec = np.ascontiguousarray(eval_records, np.float32)
    cnt = np.ascontiguousarray(count, np.int32)
    msk = None if role_mask is None else np.ascontiguousarray(role_mask, np.uint8)
    if msk is not None and msk.shape != cnt.shape:
        raise ValueError('role_mask must have one entry per agent')
    if srec.shape != erec.shape:
        raise ValueError('the safety records and the tracker records must have the same shape')
    wc = cfg.num_worlds - world_begin if world_count is None else int(world_count)
    out = np.zeros((wc, SAFETY_NPARTIALS) if msk is None else (wc, 2, SAFETY_NPARTIALS), np.float64)
    _lib.check(_lib.load().rlca_safety_reduce_host(C.byref(cfg), vp(srec), vp(erec), vp(cnt), vp(msk), srec.shape[1],
                                                   int(world_begin), wc, vp(out)))
    return out


def safety_totals(partials):
    """Per-world safety partials (rows in global world order): every column summed left to right except the last,
    'min_separation', which is the minimum of the rows; the same bits however the rows were sharded."""
    p = np.asarray(partials, np.float64).reshape(-1, SAFETY_NPARTIALS)
    tot = np.zeros(SAFETY_NPARTIALS, np.float64)
    tot[-1] = math.inf
    for row in p:
        tot[:-1] = tot[:-1] + row[:-1]
        tot[-1] = min(tot[-1], row[-1])
    return tot


def safety_metrics(tot):
    """Crashes by cause (counts, and shares of the crashes), and over the episodes that reached the goal the mean and
    population std of the minimum separation and the minimum clearance (over those where it is finite), the share with
    a near-miss tick and the mean near-miss ticks; 'min_separation' is the least of all recorded episodes."""
    t = dict(zip(SAFETY_COLUMNS, np.asarray(tot, np.float64).tolist()))
    crashes = t['crash_static'] + t['crash_robot']
    n = t['reached']
    out = {k: int(t[k]) for k in ('crash_static', 'crash_robot', 'crash_both_in_range', 'crash_into_masked', 'reached',
                                  'near_episodes')}
    out['crash_robot_share'] = t['crash_robot'] / crashes if crashes else math.nan
    for name, cnt, col in (('min_separation_reached', 'reached_separation', 'separation'),
                           ('min_clearance_reached', 'reached_clearance', 'clearance')):
        k = t[cnt]
        if k:
            mean = t['sum_' + col] / k
            out[name] = (mean, math.sqrt(max(t['sum_' + col + '_sq'] / k - mean * mean, 0.0)))
        else:
            out[name] = (math.nan, math.nan)
    out['near_miss_rate'] = t['near_episodes'] / n if n else math.nan
    out['mean_near_miss_ticks'] = t['sum_near_ticks'] / n if n else math.nan
    out['min_separation'] = t['min_separation']
    return out


def progress_params(params=None):
    """_lib.ProgressParams from a dict of any of PROGRESS_DEFAULTS' keys (the others take their defaults); ValueError
    unless window is an integer >= 1 and the distances are finite and >= 0."""
    p = dict(PROGRESS_DEFAULTS)
    unknown = set(params or ()) - set(p)
    if unknown:
        raise ValueError(f'unknown progress parameters: {sorted(unknown)}')
    p.update(params or {})
    if int(p['window']) != p['window'] or int(p['window']) < 1:
        raise ValueError('window must be an integer >= 1')
    for k in ('progress_dist', 'still_dist', 'block_dist'):
        if not (math.isfinite(float(p[k])) and float(p[k]) >= 0.0):
            raise ValueError(f'{k} must be finite and >= 0')
    return _lib.ProgressParams(int(p['window']), float(p['progress_dist']), float(p['still_dist']),
                               float(p['block_dist']))


class ProgressTracker:
    """Per-episode progress records next to an EpisodeTracker's (DESIGN.md §9o): closest distance to the goal, ticks
    since the last `progress_dist` of progress, still ticks (centre moved less than `still_dist`), rotation, whether
    another robot stood within `block_dist`, and the cause of a time-out: frozen, stalled or slow, + 4 with a robot
    near.  `params` is a dict of any of PROGRESS_DEFAULTS' keys.  Call `track()` after each `env.control_vel` and
    BEFORE `tracker.track()`: the episode a tick belongs to and the record slot are read from the tracker's state as
    its own call will see them."""

    def __init__(self, env, tracker, params=None):
        self._params = progress_params(params)
        self.params = dict(PROGRESS_DEFAULTS, **(params or {}))
        self.env, self.tracker = env, tracker
        N, E, dev = env.N, tracker.episodes, env.device
        self.running = torch.zeros(N, 4, device=dev)
        self.counters = torch.zeros(N, 4, dtype=torch.int32, device=dev)
        self.records = torch.zeros(N, E, 4, device=dev)
        self.causes = torch.zeros(N, E, dtype=torch.uint8, device=dev)
        self._st = _lib.ProgressState(_ptr(self.running), _ptr(self.counters), _ptr(self.records), _ptr(self.causes),
                                      E)

    def reset(self):
        """Forget every record and the running episodes (with the tracker's own reset())."""
        for t in (self.running, self.counters, self.records, self.causes):
            t.zero_()

    def track(self):
        """Progress records of the tick `env.control_vel` just ran (same stream, no synchronisation)."""
        env = self.env
        if not env._ticked:
            raise RuntimeError('ProgressTracker.track() needs a tick: call env.control_vel first')
        s_in, s_out = env._state_struct(1 - env._cur), env._state_struct(env._cur)
        io = env._io(action=env._keep[0], out=env._last_out)
        _lib.check(env.lib.rlca_progress_track(C.byref(env.cfg), C.byref(self._params), C.byref(s_in),
                                               C.byref(s_out), C.byref(io), C.byref(self.tracker._st),
                                               C.byref(self._st), env._stream()))

    def partials(self, world_begin=0, world_count=None, role_mask=None):
        """(world_count, PROGRESS_NPARTIALS) float64 per-world partials, or (world_count, 2, PROGRESS_NPARTIALS) split
        by the agent mask `role_mask` (N): row 0 over the agents with mask 0, row 1 over the others."""
        env = self.env
        wc = env.num_worlds - world_begin if world_count is None else int(world_count)
        m = None
        if role_mask is not None:
            m = torch.as_tensor(role_mask, device=env.device).to(torch.uint8).contiguous()
            if m.shape != (env.N,):
                raise ValueError(f'role_mask must have ({env.N},) entries')
        shape = (wc, PROGRESS_NPARTIALS) if m is None else (wc, 2, PROGRESS_NPARTIALS)
        out = torch.empty(shape, dtype=torch.float64, device=env.device)
        _lib.check(env.lib.rlca_progress_reduce(C.byref(env.cfg), C.byref(self._params), C.byref(self._st),
                                                C.byref(self.tracker._st), _ptr(m), int(world_begin), wc, _ptr(out),
                                                env._stream()))
        return out.cpu().numpy()


def progress_track_host(cfg, params, pose_in, meta_in, pose_out, flags, closed, count, state):
    """rlca_progress_track on host arrays (the same code, run by the CPU).  `params` as ProgressTracker's; `state` is a
    dict of running (N, 4) float32, counters (N, 4) int32, records (N, E, 4) float32 and causes (N, E) uint8, updated
    in place."""
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    for k, dt in (('running', np.float32), ('counters', np.int32), ('records', np.float32), ('causes', np.uint8)):
        if state[k].dtype != dt or not state[k].flags.c_contiguous:
            raise ValueError(f'state[{k!r}] must be a contiguous {np.dtype(dt).name} array')
    args = [np.ascontiguousarray(pose_in, np.float32), np.ascontiguousarray(meta_in, np.int32),
            np.ascontiguousarray(pose_out, np.float32), np.ascontiguousarray(flags, np.uint8),
            np.ascontiguousarray(closed, np.int32), np.ascontiguousarray(count, np.int32)]
    _lib.check(_lib.load().rlca_progress_track_host(
        C.byref(cfg), C.byref(progress_params(params)), *(vp(a) for a in args), state['records'].shape[1],
        *(vp(state[k]) for k in ('running', 'counters', 'records', 'causes'))))
    return state


def progress_reduce_host(cfg, params, state, eval_records, count, open_, role_mask=None, world_begin=0,
                         world_count=None):
    """rlca_progress_reduce on host arrays (`state` as progress_track_host's; the tracker's records, count and open):
    (world_count, PROGRESS_NPARTIALS), or (world_count, 2, ...) with a mask."""
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    prec = np.ascontiguousarray(state['records'], np.float32)
    causes = np.ascontiguousarray(state['causes'], np.uint8)
    running = np.ascontiguousarray(state['running'], np.float32)
    counters = np.ascontiguousarray(state['counters'], np.int32)
    erec = np.ascontiguousarray(eval_records, np.float32)
    cnt = np.ascontiguousarray(count, np.int32)
    opn = np.ascontiguousarray(open_, np.int32)
    msk = None if role_mask is None else np.ascontiguousarray(role_mask, np.uint8)
    if msk is not None and msk.shape != cnt.shape:
        raise ValueError('role_mask must have one entry per agent')
    if prec.shape != erec.shape or causes.shape != prec.shape[:2]:
        raise ValueError('the progress records, causes and the tracker records must have matching shapes')
    wc = cfg.num_worlds - world_begin if world_count is None else int(world_count)
    out = np.zeros((wc, PROGRESS_NPARTIALS) if msk is None else (wc, 2, PROGRESS_NPARTIALS), np.float64)
    _lib.check(_lib.load().rlca_progress_reduce_host(
        C.byref(cfg), C.byref(progress_params(params)), vp(prec), vp(causes), vp(running), vp(counters), vp(erec),
        vp(cnt), vp(opn), vp(msk), prec.shape[1], int(world_begin), wc, vp(out)))
    return out


def progress_totals(partials):
    """Per-world progress partials (rows in global world order) summed left to right: the same bits however the rows
    were sharded."""
    p = np.asarray(partials, np.float64).reshape(-1, PROGRESS_NPARTIALS)
    tot = np.zeros(PROGRESS_NPARTIALS, np.float64)
    for row in p:
        tot = tot + row
    return tot


def progress_metrics(tot):
    """For the time-outs and for the unfinished episodes: their number, the counts and shares of each cause (frozen,
    stalled, slow) and of those with a robot near, and the mean and population std of the closest distance to the
    goal (over those with a folded tick); the share of still ticks among all ticks of the recorded episodes; the mean
    and std of the rotation of the episodes that reached the goal.  NaN where there is nothing to average."""
    t = dict(zip(PROGRESS_COLUMNS, np.asarray(tot, np.float64).tolist()))
    ms = lambda s, s2, n: (s / n, math.sqrt(max(s2 / n - (s / n) ** 2, 0.0))) if n else (math.nan, math.nan)
    out = {}
    for g, count in (('timeout', 'timeouts'), ('unfinished', 'unfinished')):
        n = t[g + '_frozen'] + t[g + '_stalled'] + t[g + '_slow']
        out[count] = int(n)
        for k in ('frozen', 'stalled', 'slow', 'robot_near'):
            out[g + '_' + k] = int(t[g + '_' + k])
            out[g + '_' + k + '_share'] = t[g + '_' + k] / n if n else math.nan
        out[g + '_closest'] = ms(t[g + '_sum_closest'], t[g + '_sum_closest_sq'], t[g + '_folded'])
    out['still_share'] = t['sum_still_ticks'] / t['sum_ticks'] if t['sum_ticks'] else math.nan
    out['reached'] = int(t['reached'])
    out['rotation_reached'] = ms(t['sum_rotation'], t['sum_rotation_sq'], t['reached'])
    return out


def non_cooperative_mask(robots_per_world, num_worlds, k):
    """(robots_per_world * num_worlds,) uint8 with robots floor(j R / k), j < k, of every world set: k robots spread
    evenly round the circle table (DESIGN.md §9h).  ValueError unless 1 <= k <= R."""
    R, W, k = int(robots_per_world), int(num_worlds), int(k)
    if not 1 <= k <= R:
        raise ValueError(f'the number of non-cooperative robots must be in 1..{R}, got {k}')
    m = np.zeros((W, R), np.uint8)
    m[:, [j * R // k for j in range(k)]] = 1
    return m.reshape(-1)


def totals(partials):
    """Per-world partials (rows in global world order) summed left to right: the same bits however the rows were
    sharded."""
    p = np.asarray(partials, np.float64).reshape(-1, NPARTIALS)
    tot = np.zeros(NPARTIALS, np.float64)
    for row in p:
        tot = tot + row
    return tot


def metrics(tot):
    """Rates over ended episodes; mean and population std of travel time, extra time, extra distance and average
    speed over the episodes that reached the goal (NaN when there are none)."""
    t = dict(zip(COLUMNS, np.asarray(tot, np.float64).tolist()))
    ended = t['reached'] + t['crashed'] + t['timed_out']
    n = t['reached']
    rate = lambda k: t[k] / ended if ended else math.nan
    out = {'episodes': int(ended), 'reached': int(n), 'crashed': int(t['crashed']), 'timed_out': int(t['timed_out']),
           'unfinished': int(t['unfinished']), 'success_rate': rate('reached'), 'crash_rate': rate('crashed'),
           'timeout_rate': rate('timed_out')}
    for name, col in (('travel_time', 'time'), ('extra_time', 'extra_time'), ('extra_distance', 'extra_distance'),
                      ('average_speed', 'speed')):
        if n:
            mean = t['sum_' + col] / n
            var = max(t['sum_' + col + '_sq'] / n - mean * mean, 0.0)
            out[name] = (mean, math.sqrt(var))
        else:
            out[name] = (math.nan, math.nan)
    out['mean_straight_distance'] = t['sum_straight'] / n if n else math.nan
    return out


def per_arena(partials, layout, world_offset=0):
    """evaluate()'s per-world partials (rows in world order from global world `world_offset`) grouped by arena with
    pick 0's rule, world w in arena (world_offset + w) mod T (DESIGN.md §9z): one dict per arena a = 0 .. T-1 with
    'arena', 'cells' (its placeable cells), 'worlds', 'totals' (totals of its rows) and 'metrics' (metrics of those)."""
    p = np.asarray(partials, np.float64).reshape(-1, NPARTIALS)
    T = int(layout.count)
    arena = (int(world_offset) + np.arange(len(p))) % T
    cells = np.diff(np.asarray(layout.tables.cell_off, np.int64))
    out = []
    for a in range(T):
        tot = totals(p[arena == a])
        out.append({'arena': a, 'cells': int(cells[a]), 'worlds': int((arena == a).sum()), 'totals': tot,
                    'metrics': metrics(tot)})
    return out


def evaluate(env, policy, episodes, max_ticks, check_every=50, non_cooperative=None, hybrid=None, safety=None,
             progress=None, noise=None, latency=None, dynamics=None, localization=None, crowd=None, planner=None):
    """Drive every agent of `env` with the deterministic mean action of `policy` (generate_action_no_sampling, scans
    through the env's FIFO), or with the actions of `policy` when it is an OrcaController or NhOrcaController (orca.py, map-blind or map-aware), until each has `episodes` recorded episodes or `max_ticks` ticks have run, and reduce
    the records.  The episode mechanics are the env's: auto_reset 1 (stage 1) and 2 (stage 2) re-spawn inside the
    tick; auto_reset 0 (circle) runs one episode per robot: a robot that was terminal on the previous tick gets v = 0
    and its first termination is the record, so at most one record per robot.  Robots that hold all their records keep
    driving: they are obstacles for the others.  Completion is checked every `check_every` ticks (one sync each).
    On a scenario with a random layout (make_scenario('random') or 'arena') every world first draws its own starts and
    goals (env.random_layout).  Returns {'partials', 'totals', 'metrics', 'ticks', 'tracker'}.

    With `non_cooperative` (an orca.NonCooperative on `env`) its robots drive straight to their goals instead: the
    override is applied to every tick's action before the circle rule, so they keep the same episode mechanics.  The
    result then also holds 'partials_split' (num_worlds, 2, NPARTIALS) and 'by_role' {'cooperative',
    'non_cooperative'}: the metrics of each role; 'partials', 'totals' and 'metrics' still cover every robot.

    With `hybrid` (an orca.Hybrid on `env`, policies only) the policy's action is switched per robot by its newest scan
    before the non-cooperative override, so masked robots still get the driver's action.  The result then also holds
    'mode_counts' (num_worlds, 3) int64, the ticks of tracked episodes each world's robots spent in each mode, and
    'modes' (orca.mode_shares: the share of those agent-ticks per mode and 'agent_ticks'); with `non_cooperative`
    both cover the cooperative robots only.

    With `safety` (a near-miss distance in metres) a SafetyTracker runs before the episode tracker on every tick and
    the result also holds 'safety_partials' (num_worlds, SAFETY_NPARTIALS), 'safety_totals', 'safety'
    (safety_metrics) and 'safety_tracker'; with `non_cooperative` also 'safety_partials_split' and 'safety_by_role',
    where the cooperative row's 'crash_into_masked' counts its crashes into a non-cooperative robot.  With None nothing
    of this is allocated or launched.

    With `progress` (a dict of any of PROGRESS_DEFAULTS' keys, {} for the defaults) a ProgressTracker runs before the
    episode tracker on every tick and the result also holds 'progress_partials' (num_worlds, PROGRESS_NPARTIALS),
    'progress_totals', 'progress' (progress_metrics) and 'progress_tracker'; with `non_cooperative` also
    'progress_partials_split' and 'progress_by_role'.  With None nothing of this is allocated or launched.

    With `noise`, `latency`, `dynamics` or `localization` (a noise.Noise, latency.Latency, dynamics.Dynamics or
    localization.Localization on `env`, DESIGN.md §9p-§9s) the robots sense and act through a perturbation.Chain of
    them, which fixes their order (§9y): the command, after the masked override and the circle rule, becomes the
    chain's executed command, and the first stack and every stack a tick wrote are perturbed before the policy reads
    them.  A circle robot stopped by the circle rule still runs out its queued commands and brakes at its limit.
    env.obs, env.gs and the state are never perturbed, so the trackers keep measuring the truth.  The result then also
    holds each one's settings under its name.  Scan noise and scan delay need a policy: the ORCA baselines do not read
    the scan.  The ORCA baselines command velocities like the policy, so command latency, actuation noise and the
    limits apply to them.  Localization error is for policies only, not hybrid: the ORCA baselines and the hybrid
    driver read the true state through their own kernels; non-cooperative robots keep the truth.

    With `crowd` (a crowd.Crowd on `env`, DESIGN.md §9t) its agents follow the social force instead, applied where the
    non-cooperative override is, and the result holds the same role splits with the keys 'cooperative' and 'crowd'
    (mode counts over the cooperative robots likewise).  Crowd agents read the true state.  ValueError together with
    `non_cooperative`: the split has two roles.

    With `policy` a dwa.DwaController on `env` (DESIGN.md §9u) every robot is driven by the dynamic-window baseline,
    which reads what the policy would: on each tick it is called with the stack the policy would read and the gs under
    localization, env.gs otherwise.  Everything after it is the policy's chain: the masked override, the circle rule,
    latency, noise and dynamics, so every sensing perturbation applies to it.  The result then also holds 'dwa' (the
    settings and 'fallback_share': the robot-ticks, over all robot-ticks, on which no candidate was admissible and it
    commanded (0, 0)).  ValueError together with `hybrid`, which switches a policy.

    With `planner` (a planner.Planner on `env`, DESIGN.md §9w), the chain's last link, the planner is updated at the
    start and after every tick, before the trackers: it re-plans the robots whose goal changed and keeps every
    episode's geodesic length.  With planner.steer the policy (or the DWA baseline) reads the
    planner's gs: a waypoint on the geodesic path as the local goal where the goal is out of sight.  The result then
    also holds 'geodesic_partials' (num_worlds, planner.NPARTIALS), 'geodesic_totals' and 'geodesic'
    (planner.geodesic_metrics), with `non_cooperative` or `crowd` also 'geodesic_partials_split' and
    'geodesic_by_role'; with steer also 'planner': the settings and the share of robot-ticks of the cooperative robots
    with each status (goal visible, waypoint, no plan).  Without steer it works with every controller.  ValueError for
    steer with the ORCA baselines or `hybrid` (they read the true goal) and with `localization` (the planner plans from
    the true pose)."""
    dwa = isinstance(policy, DwaController)
    orca = isinstance(policy, (OrcaController, NhOrcaController))
    if dwa:
        if policy.env is not env:
            raise ValueError('the DWA controller belongs to another env')
        if hybrid is not None:
            raise ValueError('hybrid switches a policy; the DWA baseline is not switched')
    if crowd is not None:
        if non_cooperative is not None:
            raise ValueError('crowd and non_cooperative cannot be combined: the metrics split into two roles')
        if crowd.env is not env:
            raise ValueError('the crowd belongs to another env')
    masked, role = (crowd, 'crowd') if crowd is not None else (non_cooperative, 'non_cooperative')
    chain = Chain(env, noise, latency, dynamics, localization, planner)
    if localization is not None:
        if orca:
            raise ValueError('localization error changes what a policy reads; the ORCA baselines read the true state')
        if hybrid is not None:
            raise ValueError('localization error changes what a policy reads; the hybrid driver reads the true state')
    if planner is not None and planner.steer:
        if orca:
            raise ValueError('the planner steers what a policy reads; the ORCA baselines read the true goal through '
                             'their own kernels')
        if hybrid is not None:
            raise ValueError('the planner steers what a policy reads; the hybrid driver reads the true goal')
    if latency is not None and latency.params.scan_on and orca:
        raise ValueError('scan delay changes what a policy reads; the ORCA baselines do not read the scan')
    E = int(episodes)
    if int(check_every) < 1:
        raise ValueError('check_every must be >= 1')
    if hybrid is not None and orca:
        raise ValueError('hybrid switches a policy; the ORCA baselines are not switched')
    if noise is not None and noise.params.scan_on and orca:
        raise ValueError('scan noise perturbs what a policy reads; the ORCA baselines do not read the scan')
    tracker = EpisodeTracker(env, E)
    safe = SafetyTracker(env, tracker, safety) if safety is not None else None
    prog = ProgressTracker(env, tracker, progress) if progress is not None else None
    N, dev = env.N, env.device
    circle = int(env.cfg.auto_reset) == 0
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    if env.sc.layout is not None:
        env.random_layout()
    tracker.reset()
    if hybrid is not None:
        hybrid.reset()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(N, 3, env.beam_mum, device=dev)]
    if planner is not None:
        planner.attach(tracker)
    gs = chain.sense(stacks[0])
    terminal = torch.zeros(N, dtype=torch.bool, device=dev)
    fallbacks = torch.zeros(N, dtype=torch.int64, device=dev) if dwa else None
    goal_done = 1 if circle else E
    ticks = 0
    for tick in range(int(max_ticks)):
        k = tick & 1
        if orca:
            scaled = policy()
        elif dwa:
            scaled = policy(stacks[k], env.gs if gs is None else gs)
            fallbacks += policy.status()
        else:
            goal, speed = (env.get_local_goal(), env.get_self_speed()) if gs is None else (gs[:, 0:2], gs[:, 2:4])
            _, scaled = generate_action_no_sampling(env=env, state_list=(stacks[k], goal, speed), policy=policy,
                                                    action_bound=ACTION_BOUND)
            if hybrid is not None:
                hybrid.apply(scaled, stacks[k], tracker)
        if masked is not None:
            masked.apply(scaled)
        if circle:
            scaled = torch.stack((torch.where(terminal, 0.0, scaled[:, 0]), scaled[:, 1]), 1)
        scaled = chain.command(scaled, env.flags if tick > 0 else None)
        env.control_vel(scaled, stack_in=stacks[k], stack_out=stacks[1 - k])
        gs = chain.sense(stacks[1 - k], env.flags)
        if safe is not None:
            safe.track()
        if prog is not None:
            prog.track()
        tracker.track()
        if circle:
            terminal = env.flags[:, 0] != 0
        ticks = tick + 1
        if ticks % check_every == 0 and bool((tracker.count >= goal_done).all()):
            break
    part = tracker.partials()
    tot = totals(part)
    out = {'partials': part, 'totals': tot, 'metrics': metrics(tot), 'ticks': ticks, 'tracker': tracker}
    if masked is not None:
        split = tracker.partials_split(masked.mask)
        out['partials_split'] = split
        out['by_role'] = {'cooperative': metrics(totals(split[:, 0])),
                          role: metrics(totals(split[:, 1]))}
    if hybrid is not None:
        out['mode_counts'] = hybrid.counts_per_world(None if masked is None else masked.mask)
        out['modes'] = mode_shares(out['mode_counts'])
    if safe is not None:
        sp = safe.partials()
        out.update(safety_partials=sp, safety_totals=safety_totals(sp), safety_tracker=safe)
        out['safety'] = safety_metrics(out['safety_totals'])
        if masked is not None:
            ss = safe.partials(role_mask=masked.mask)
            out['safety_partials_split'] = ss
            out['safety_by_role'] = {'cooperative': safety_metrics(safety_totals(ss[:, 0])),
                                     role: safety_metrics(safety_totals(ss[:, 1]))}
    if prog is not None:
        pp = prog.partials()
        out.update(progress_partials=pp, progress_totals=progress_totals(pp), progress_tracker=prog)
        out['progress'] = progress_metrics(out['progress_totals'])
        if masked is not None:
            ps = prog.partials(role_mask=masked.mask)
            out['progress_partials_split'] = ps
            out['progress_by_role'] = {'cooperative': progress_metrics(progress_totals(ps[:, 0])),
                                       role: progress_metrics(progress_totals(ps[:, 1]))}
    if planner is not None:
        gp = planner.partials()
        out.update(geodesic_partials=gp, geodesic_totals=geodesic_totals(gp))
        out['geodesic'] = geodesic_metrics(out['geodesic_totals'])
        if masked is not None:
            gsp = planner.partials(role_mask=masked.mask)
            out['geodesic_partials_split'] = gsp
            out['geodesic_by_role'] = {'cooperative': geodesic_metrics(geodesic_totals(gsp[:, 0])),
                                       role: geodesic_metrics(geodesic_totals(gsp[:, 1]))}
        if planner.steer:
            out['planner'] = dict(planner.settings(),
                                  **planner.status_shares(None if masked is None else masked.mask))
    out.update(chain.settings())
    if dwa:
        out['dwa'] = dict(policy.settings(), fallback_share=int(fallbacks.sum()) / (ticks * N) if ticks else math.nan)
    return out
