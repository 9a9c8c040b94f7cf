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
from .model.ppo import generate_action_no_sampling
from .orca import NhOrcaController, OrcaController

COLUMNS = _lib.EVAL_PARTIALS
NPARTIALS = len(COLUMNS)
ACTION_BOUND = [[0, -1], [1, 1]]
# the reference's episode mechanics per scenario: stage 1 re-spawns a robot as soon as it is done
# (ppo_stage1.py:51-65), stage 2 re-spawns a group when all of it is done (ppo_stage2.py:49-106), circle runs one
# episode that the caller never resets (circle_test.py:36-84)
AUTO_RESET = {'stage1': 1, 'stage2': 2, 'circle': 0}


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


def evaluate(env, policy, episodes, max_ticks, check_every=50):
    """Drive every agent of `env` with the deterministic mean action of `policy` (generate_action_no_sampling, scans
    through the env's FIFO), or with the actions of `policy` when it is an OrcaController or NhOrcaController (orca.py, map-blind or map-aware), until each has `episodes` recorded episodes or `max_ticks` ticks have run, and reduce
    the records.  The episode mechanics are the env's: auto_reset 1 (stage 1) and 2 (stage 2) re-spawn inside the
    tick; auto_reset 0 (circle) runs one episode per robot: a robot that was terminal on the previous tick gets v = 0
    and its first termination is the record, so at most one record per robot.  Robots that hold all their records keep
    driving: they are obstacles for the others.  Completion is checked every `check_every` ticks (one sync each).
    Returns {'partials', 'totals', 'metrics', 'ticks', 'tracker'}."""
    E = int(episodes)
    if int(check_every) < 1:
        raise ValueError('check_every must be >= 1')
    tracker = EpisodeTracker(env, E)
    N, dev = env.N, env.device
    circle = int(env.cfg.auto_reset) == 0
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    tracker.reset()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(N, 3, env.beam_mum, device=dev)]
    terminal = torch.zeros(N, dtype=torch.bool, device=dev)
    goal_done = 1 if circle else E
    ticks = 0
    for tick in range(int(max_ticks)):
        k = tick & 1
        if isinstance(policy, (OrcaController, NhOrcaController)):
            scaled = policy()
        else:
            _, scaled = generate_action_no_sampling(env=env, state_list=(stacks[k], env.get_local_goal(),
                                                                         env.get_self_speed()),
                                                    policy=policy, action_bound=ACTION_BOUND)
        if circle:
            scaled = torch.stack((torch.where(terminal, 0.0, scaled[:, 0]), scaled[:, 1]), 1)
        env.control_vel(scaled, stack_in=stacks[k], stack_out=stacks[1 - k])
        tracker.track()
        if circle:
            terminal = env.flags[:, 0] != 0
        ticks = tick + 1
        if ticks % check_every == 0 and bool((tracker.count >= goal_done).all()):
            break
    part = tracker.partials()
    tot = totals(part)
    return {'partials': part, 'totals': tot, 'metrics': metrics(tot), 'ticks': ticks, 'tracker': tracker}
