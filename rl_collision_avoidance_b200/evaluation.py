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
from .orca import NhOrcaController, OrcaController, mode_shares

COLUMNS = _lib.EVAL_PARTIALS
NPARTIALS = len(COLUMNS)
ACTION_BOUND = [[0, -1], [1, 1]]
# the reference's episode mechanics per scenario: stage 1 re-spawns a robot as soon as it is done
# (ppo_stage1.py:51-65), stage 2 re-spawns a group when all of it is done (ppo_stage2.py:49-106), circle runs one
# episode that the caller never resets (circle_test.py:36-84); so does the random scenario, one layout per world
AUTO_RESET = {'stage1': 1, 'stage2': 2, 'circle': 0, 'random': 0}


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


def evaluate(env, policy, episodes, max_ticks, check_every=50, non_cooperative=None, hybrid=None):
    """Drive every agent of `env` with the deterministic mean action of `policy` (generate_action_no_sampling, scans
    through the env's FIFO), or with the actions of `policy` when it is an OrcaController or NhOrcaController (orca.py, map-blind or map-aware), until each has `episodes` recorded episodes or `max_ticks` ticks have run, and reduce
    the records.  The episode mechanics are the env's: auto_reset 1 (stage 1) and 2 (stage 2) re-spawn inside the
    tick; auto_reset 0 (circle) runs one episode per robot: a robot that was terminal on the previous tick gets v = 0
    and its first termination is the record, so at most one record per robot.  Robots that hold all their records keep
    driving: they are obstacles for the others.  Completion is checked every `check_every` ticks (one sync each).
    On a scenario with a random layout (make_scenario('random')) every world first draws its own starts and goals
    (env.random_layout).  Returns {'partials', 'totals', 'metrics', 'ticks', 'tracker'}.

    With `non_cooperative` (an orca.NonCooperative on `env`) its robots drive straight to their goals instead: the
    override is applied to every tick's action before the circle rule, so they keep the same episode mechanics.  The
    result then also holds 'partials_split' (num_worlds, 2, NPARTIALS) and 'by_role' {'cooperative',
    'non_cooperative'}: the metrics of each role; 'partials', 'totals' and 'metrics' still cover every robot.

    With `hybrid` (an orca.Hybrid on `env`, policies only) the policy's action is switched per robot by its newest scan
    before the non-cooperative override, so masked robots still get the driver's action.  The result then also holds
    'mode_counts' (num_worlds, 3) int64, the ticks of tracked episodes each world's robots spent in each mode, and
    'modes' (orca.mode_shares: the share of those agent-ticks per mode and 'agent_ticks'); with `non_cooperative`
    both cover the cooperative robots only."""
    E = int(episodes)
    if int(check_every) < 1:
        raise ValueError('check_every must be >= 1')
    if hybrid is not None and isinstance(policy, (OrcaController, NhOrcaController)):
        raise ValueError('hybrid switches a policy; the ORCA baselines are not switched')
    tracker = EpisodeTracker(env, E)
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
            if hybrid is not None:
                hybrid.apply(scaled, stacks[k], tracker)
        if non_cooperative is not None:
            non_cooperative.apply(scaled)
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
    out = {'partials': part, 'totals': tot, 'metrics': metrics(tot), 'ticks': ticks, 'tracker': tracker}
    if non_cooperative is not None:
        split = tracker.partials_split(non_cooperative.mask)
        out['partials_split'] = split
        out['by_role'] = {'cooperative': metrics(totals(split[:, 0])),
                          'non_cooperative': metrics(totals(split[:, 1]))}
    if hybrid is not None:
        out['mode_counts'] = hybrid.counts_per_world(None if non_cooperative is None else non_cooperative.mask)
        out['modes'] = mode_shares(out['mode_counts'])
    return out
