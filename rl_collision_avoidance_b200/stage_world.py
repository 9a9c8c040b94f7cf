"""Batched `StageWorld`: the reference's env-client surface over the fused CUDA tick.

Mirrors `class StageWorld` of /root/reference/stage_world1.py:16-274 (and the
stage2 / circle variants) method for method, but ONE object holds the whole
agent batch (`num_worlds` independent worlds x `num_env` robots each) and every
method returns device tensors with a leading agent axis N = num_worlds*num_env:

    reference (per robot)                     here (batched)
    get_laser_observation() -> (beam,)        (N, beam) f32           stage_world1.py:122-140
    get_local_goal()        -> [x, y]         (N, 2)                  :155-160
    get_self_speed()        -> [v, w]         (N, 2)                  :143-144
    get_self_stateGT()      -> [x, y, th]     (N, 3)                  :116-117
    get_crash_state()       -> 0/1            (N,) u8                 :149-150
    control_vel(action)                       action (N, 2); runs the tick      :226-234
    get_reward_and_terminate(t) -> (r, terminate, result)
                                              (N,) f32, (N,) bool, (N,) u8 code :180-211
    reset_world / reset_pose / generate_goal_point                  :162-177,213-223

Result codes: 0 none, 1 'Reach Goal', 2 'Crashed', 3 'Time out'.
`reset()` and `step(action)` are conveniences named by BASELINE.json.

ROS topics, the stageros bridge and mpi4py gather/scatter are gone: the batch is
already "gathered" on the device.  All compute is in librlca.so (hand-written
sm_90a CUDA behind the C ABI of include/rlca.h); torch only owns the memory.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .scenarios import ArenaLayout, Scenario, arena_tables_struct, fill_config, make_scenario

RESULT_STRINGS = {0: 0, 1: 'Reach Goal', 2: 'Crashed', 3: 'Time out'}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class StageWorld:
    def __init__(self, beam_num, index=0, num_env=None, *, scenario='stage1', num_worlds=1, device='cuda:0',
                 seed=0, auto_reset=False, world_offset=0, raw_beams=None, map=None, ctas_per_world=0,
                 max_reject=4096):
        if not torch.cuda.is_available():
            raise _lib.RlcaError('StageWorld needs a CUDA device: the simulator has no CPU path')
        self.lib = _lib.load()
        self.index = index                     # kept: generate_action branches on env.index == 0 (model/ppo.py:58)
        self.device = torch.device(device)
        self.sc: Scenario = scenario if isinstance(scenario, Scenario) else make_scenario(scenario, map, num_env)
        if num_env is not None and num_env != self.sc.robots_per_world:
            raise ValueError(f'scenario {self.sc.name} has {self.sc.robots_per_world} robots per world, got num_env={num_env}')
        self.num_env = self.sc.robots_per_world
        self.num_worlds = int(num_worlds)
        self.beam_mum = int(beam_num)           # (sic) the reference's attribute name, stage_world1.py:23
        self.N = self.num_env * self.num_worlds
        self.cfg = fill_config(_lib.EnvConfig(), self.sc, num_worlds=self.num_worlds, beams=self.beam_mum,
                               raw_beams=raw_beams, auto_reset=auto_reset, seed=seed, world_offset=world_offset,
                               max_reject=max_reject)
        torch.cuda.set_device(self.device)
        h = C.c_void_p()
        _lib.check(self.lib.rlca_env_create(C.byref(self.cfg), C.byref(h)))
        self._h = h
        cells = np.ascontiguousarray(self.sc.map.cells, dtype=np.uint8)
        _lib.check(self.lib.rlca_env_set_map(self._h, cells.ctypes.data_as(C.c_void_p), cells.shape[1], cells.shape[0]))
        it = np.ascontiguousarray(self.sc.init_tab, dtype=np.float32)
        gt = np.ascontiguousarray(self.sc.goal_tab, dtype=np.float32)
        _lib.check(self.lib.rlca_env_set_tables(self._h, it.ctypes.data_as(C.c_void_p), gt.ctypes.data_as(C.c_void_p)))
        if ctas_per_world:
            _lib.check(self.lib.rlca_env_set_ctas_per_world(self._h, int(ctas_per_world)))
        N, dev = self.N, self.device
        # ping-pong simulator state (see rlca_env_step: several CTAs read one world's robots)
        self._st = [dict(pose=torch.zeros(N, 4, device=dev), goal=torch.zeros(N, 4, device=dev),
                         acc=torch.zeros(N, 4, device=dev), meta=torch.zeros(N, 4, dtype=torch.int32, device=dev))
                    for _ in range(2)]
        self._cur = 0
        self.obs = torch.zeros(N, self.beam_mum, device=dev)
        self.reward = torch.zeros(N, device=dev)
        self.flags = torch.zeros(N, 4, dtype=torch.uint8, device=dev)
        self.gs = torch.zeros(N, 4, device=dev)
        self.eplog = torch.zeros(N, 8, device=dev)
        self._action = torch.zeros(N, 2, device=dev)
        self._host = None
        self._host_ptrs = None
        self._ticked = False
        if self.sc.layout is not None:
            # training on random layouts (relayout_finished): the next tick's live mask and the per-world status
            self.live = torch.ones(N, dtype=torch.uint8, device=dev)
            self._relayout_status = torch.zeros(self.num_worlds, dtype=torch.int32, device=dev)
            self._layout_params = _lib.LayoutParams(self.sc.layout.side, self.sc.layout.separation,
                                                    self.sc.layout.min_travel)
            self._arena = None
            if isinstance(self.sc.layout, ArenaLayout):
                # the arena tables, checked on the host and uploaded once (DESIGN.md §9v)
                t = self.sc.layout.tables
                _lib.check(self.lib.rlca_arena_tables_check(C.byref(self.cfg), C.byref(arena_tables_struct(t))))
                self._arena_off = torch.from_numpy(np.ascontiguousarray(t.cell_off, np.int32)).to(dev)
                self._arena_cells = torch.from_numpy(np.ascontiguousarray(t.cells, np.int32)).to(dev)
                self._arena = arena_tables_struct(t, self._arena_off.data_ptr(), self._arena_cells.data_ptr())
        self.reset_world()

    # ------------------------------------------------------------------ plumbing
    def _state_struct(self, k):
        # the ping-pong state tensors never move: build each struct once
        cache = self.__dict__.setdefault('_state_structs', {})
        if k not in cache:
            s = self._st[k]
            cache[k] = _lib.EnvState(_ptr(s['pose']), _ptr(s['goal']), _ptr(s['acc']), _ptr(s['meta']))
        return cache[k]

    def _io(self, action=None, live=None, obs=None, stack_in=None, stack_out=None, out=None):
        o = out or {}
        return _lib.StepIO(_ptr(action if action is not None else self._action), _ptr(live),
                           _ptr(obs if obs is not None else self.obs), _ptr(o.get('reward', self.reward)),
                           _ptr(o.get('flags', self.flags)), _ptr(o.get('gs', self.gs)),
                           _ptr(o.get('eplog', self.eplog)), _ptr(stack_in), _ptr(stack_out))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @property
    def state(self):
        return self._st[self._cur]

    def close(self):
        if getattr(self, '_h', None):
            self.lib.rlca_env_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self):
        return int(self.lib.rlca_env_launch_count(self._h))

    def set_ctas_per_world(self, s):
        _lib.check(self.lib.rlca_env_set_ctas_per_world(self._h, int(s)))

    def set_host_chunks(self, k):
        """World ranges per `step_host` call (0 = library default, 1 = strictly serial)."""
        _lib.check(self.lib.rlca_env_set_host_chunks(self._h, int(k)))

    def set_host_zero_copy(self, mode):
        """`step_host` host traffic: 1 = the kernel reads actions from / mirrors all outputs to pinned host memory (no
        DMA), 2 = small buffers only (scans by DMA in world ranges), 0 = DMA copies."""
        _lib.check(self.lib.rlca_env_set_host_zero_copy(self._h, int(mode)))

    # ------------------------------------------------------------------ reference surface
    def reset_world(self):
        """reset_positions service + zeroed speeds (stage_world1.py:162-169)."""
        st = self._state_struct(self._cur)
        none = torch.zeros(self.N, dtype=torch.uint8, device=self.device)
        _lib.check(self.lib.rlca_env_reset(self._h, C.byref(st), _ptr(none), 1, self._stream()))
        self._ticked = False

    def reset_pose(self, mask=None):
        """reset_pose + generate_goal_point for the masked agents (all when None).  The goal is
        drawn in the same kernel because it depends on the new pose (stage_world1.py:262-274)."""
        st = self._state_struct(self._cur)
        m = None if mask is None else mask.to(device=self.device, dtype=torch.uint8).contiguous()
        _lib.check(self.lib.rlca_env_reset(self._h, C.byref(st), _ptr(m), 0, self._stream()))
        self._observe()

    def generate_goal_point(self, mask=None):
        """generate_goal_point (stage_world1.py:171-177): a goal for the CURRENT pose of the masked agents (all when
        None), pre_distance refreshed.  The draws are keyed by (agent, episode), so right after reset_pose this
        re-derives the goal reset_pose already drew - the reference's call order (ppo_stage1.py:51-53) is harmless."""
        st = self._state_struct(self._cur)
        m = None if mask is None else mask.to(device=self.device, dtype=torch.uint8).contiguous()
        _lib.check(self.lib.rlca_env_reset(self._h, C.byref(st), _ptr(m), 2, self._stream()))
        self._observe()

    def generate_random_goal(self):
        """(N, 2) goals generate_goal_point would set for the current poses (stage_world1.py:262-274 and the stage-2 /
        circle variants), without touching the state."""
        return self._scratch_reset(2)['goal'][:, 0:2]

    def generate_random_pose(self):
        """(N, 3) poses the next reset_pose would teleport to (stage_world1.py:251-260; table poses where the scenario
        does not randomise), without touching the state."""
        return self._scratch_reset(0)['pose'][:, 0:3]

    def _scratch_reset(self, mode):
        sc = {k: v.clone() for k, v in self.state.items()}
        st = _lib.EnvState(_ptr(sc['pose']), _ptr(sc['goal']), _ptr(sc['acc']), _ptr(sc['meta']))
        _lib.check(self.lib.rlca_env_reset(self._h, C.byref(st), _ptr(None), mode, self._stream()))
        return sc

    def random_layout(self):
        """A random layout (DESIGN.md §9i) in every world of the current state: starts, goals and headings drawn on the
        device from the scenario's Layout (rlca_layout_random) or, on an arena scenario, in the world's arena
        (rlca_layout_arena, §9v), then the scan and local goal from the new poses.  One
        synchronisation reads the per-world status; ValueError names the first world whose robots could not all be
        placed, and that world keeps its rows."""
        lay = self.sc.layout
        if lay is None:
            raise ValueError(f'scenario {self.sc.name} has no random layout')
        params = _lib.LayoutParams(lay.side, lay.separation, lay.min_travel)
        status = torch.empty(self.num_worlds, dtype=torch.int32, device=self.device)
        st = self._state_struct(self._cur)
        if self._arena is not None:
            _lib.check(self.lib.rlca_layout_arena(C.byref(self.cfg), C.byref(params), C.byref(self._arena), lay.pick,
                                                  C.byref(st), _ptr(status), self._stream()))
        else:
            _lib.check(self.lib.rlca_layout_random(C.byref(self.cfg), C.byref(params), C.byref(st), _ptr(status),
                                                   self._stream()))
        self._observe()
        self.live.fill_(1)
        self._relayout_status.zero_()
        self._raise_layout_status(status)

    def _raise_layout_status(self, status):
        bad = torch.nonzero(status).flatten().cpu()
        if len(bad):
            w = int(bad[0])
            where = ''
            if self._arena is not None:
                where = ' in its arena' + (f' {(int(self.cfg.world_offset) + w) % self.sc.layout.count}'
                                           if self.sc.layout.pick == 0 else '')
            raise ValueError(f'world {int(self.cfg.world_offset) + w}: robot {int(status[w]) - 1} not placed{where} in '
                             f'{int(self.cfg.max_reject)} tries; lower the density')

    def relayout_finished(self, stack_out, out=None):
        """After a tick of a random scenario with auto_reset 0 (DESIGN.md §9k), on the env's stream with no
        synchronisation: park the robots whose episode ended (last command 0, `live` 0), give every world whose robots
        have all ended a new layout (rlca_layout_respawn; rlca_layout_arena_respawn on arenas), scan the new state (rlca_env_observe into the env's own obs /
        gs), and make the re-laid robots' rows of stack_out (N, 3, beams) three copies of the new scan and their
        out['gs'] rows the new local goal and speed (rlca_stack_refresh).  `out` holds the 'flags' and 'gs' buffers the
        tick wrote (default the env's own); re-laid robots get flags[:, 3] (was_reset) = 1.  Pass `live` to the next
        control_vel; check_relayout() reads the status."""
        if self.sc.layout is None:
            raise ValueError(f'scenario {self.sc.name} has no random layout')
        o = out or {}
        flags, gs = o.get('flags', self.flags), o.get('gs', self.gs)
        st = self._state_struct(self._cur)
        stream = self._stream()
        if self._arena is not None:
            _lib.check(self.lib.rlca_layout_arena_respawn(C.byref(self.cfg), C.byref(self._layout_params),
                                                          C.byref(self._arena), self.sc.layout.pick, C.byref(st),
                                                          _ptr(flags), _ptr(self.live), _ptr(self._relayout_status),
                                                          stream))
        else:
            _lib.check(self.lib.rlca_layout_respawn(C.byref(self.cfg), C.byref(self._layout_params), C.byref(st),
                                                    _ptr(flags), _ptr(self.live), _ptr(self._relayout_status), stream))
        self._observe()
        _lib.check(self.lib.rlca_stack_refresh(C.byref(self.cfg), _ptr(flags), _ptr(self.obs), _ptr(self.gs),
                                               _ptr(stack_out), _ptr(gs), stream))

    def check_relayout(self):
        """One synchronisation: ValueError naming the first world a re-layout could not fill, in random_layout()'s
        wording."""
        self._raise_layout_status(self._relayout_status)

    def control_pose(self, pose, mask=None):
        """cmd_pose (stage_world1.py:237-249 -> stageros.cpp:282-296): teleport the masked agents (all when None) to
        pose (N, 3) = x, y, yaw; no collision test, stall flag untouched; the next scan is taken from the new pose."""
        p = pose.to(device=self.device, dtype=torch.float32).reshape(self.N, 3)
        th = torch.remainder(p[:, 2] + math.pi, 2 * math.pi) - math.pi          # yaw read back in (-pi, pi]
        th = torch.where(th <= -math.pi, th + 2 * math.pi, th)
        new = torch.stack((p[:, 0], p[:, 1], th), 1)
        cur = self.state['pose']
        if mask is None:
            cur[:, 0:3] = new
        else:
            m = mask.to(device=self.device).bool()
            cur[m, 0:3] = new[m]
        self._observe()

    def _observe(self, obs=None):
        st = self._state_struct(self._cur)
        io = self._io(obs=obs)
        _lib.check(self.lib.rlca_env_observe(self._h, C.byref(st), C.byref(io), self._stream()))

    def control_vel(self, action, live=None, obs_out=None, stack_in=None, stack_out=None, out=None):
        """Publish cmd_vel and advance one 0.1 s tick (stage_world1.py:226-234 + the
        rospy.sleep(0.001) of ppo_stage1.py:78).  `action` (N,2) device tensor (raw policy
        output; clipped to the action bound inside the kernel)."""
        a = action if (action.is_cuda and action.dtype == torch.float32 and action.is_contiguous()) \
            else action.to(device=self.device, dtype=torch.float32).contiguous()
        lv = None if live is None else live.to(device=self.device, dtype=torch.uint8).contiguous()
        s_in, s_out = self._state_struct(self._cur), self._state_struct(1 - self._cur)
        io = self._io(action=a, live=lv, obs=obs_out, stack_in=stack_in, stack_out=stack_out, out=out)
        self._keep = (a, lv)
        self._last_out = out or {}
        _lib.check(self.lib.rlca_env_step(self._h, C.byref(s_in), C.byref(s_out), C.byref(io), self._stream()))
        self._cur = 1 - self._cur
        self._ticked = True

    def get_reward_and_terminate(self, t=None):
        """(reward, terminate, result) of the tick just run (stage_world1.py:180-211).  The step
        counter lives on the device (state meta[:,0]); `t` is accepted for signature parity."""
        o = getattr(self, '_last_out', {})
        flags = o.get('flags', self.flags)
        return o.get('reward', self.reward), flags[:, 0].bool(), flags[:, 2]

    def get_laser_observation(self):
        return self.obs

    def get_local_goal(self):
        return self.gs[:, 0:2]

    def get_self_speed(self):
        return self.gs[:, 2:4]

    def get_self_stateGT(self):
        return self.state['pose'][:, 0:3]

    def get_self_state(self):
        return self.state['pose'][:, 0:3]

    def get_self_speedGT(self):
        """(N, 2) ground-truth speed as stageros publishes it (stage_world1.py:88-95,119-120; stageros.cpp:580-606):
        |pose - previous pose| / dt and normalize(yaw - previous yaw) / dt, teleports included.  Zero before the
        first tick.  (The tick keeps both poses: the state is ping-ponged.)"""
        if not self._ticked:
            return torch.zeros(self.N, 2, device=self.device)
        cur, prev = self._st[self._cur]['pose'], self._st[1 - self._cur]['pose']
        d = cur[:, 0:3] - prev[:, 0:3]
        a = torch.remainder(d[:, 2] + math.pi, 2 * math.pi) - math.pi
        inv_dt = 1.0 / float(self.cfg.dt)
        return torch.stack((torch.hypot(d[:, 0], d[:, 1]) * inv_dt, a * inv_dt), 1)

    def get_crash_state(self):
        return self.state['meta'][:, 2].to(torch.uint8)

    def get_sim_time(self):
        return None

    @property
    def goal_point(self):
        return self.state['goal'][:, 0:2]

    @property
    def init_pose(self):
        return self.state['acc'][:, 2:4]

    # ------------------------------------------------------------------ BASELINE.json conveniences
    def reset(self):
        self.reset_world()
        self.reset_pose()
        self.generate_goal_point()
        return self.obs, self.get_local_goal(), self.get_self_speed()

    def step(self, action, live=None, obs_out=None, stack_in=None, stack_out=None):
        self.control_vel(action, live=live, obs_out=obs_out, stack_in=stack_in, stack_out=stack_out)
        r, d, res = self.get_reward_and_terminate()
        return (self.obs if obs_out is None else obs_out), self.get_local_goal(), self.get_self_speed(), r, d, res

    def step_host(self, action_host, want_obs=True):
        """Reference-facing tick with HOST buffers: pinned action in, pinned obs/reward/flags/gs
        out, host<->device traffic and a stream sync inside the call (rlca_env_step_host)."""
        if self._host is None:
            self._host = dict(obs=torch.empty(self.N, self.beam_mum).pin_memory(),
                              reward=torch.empty(self.N).pin_memory(),
                              flags=torch.empty(self.N, 4, dtype=torch.uint8).pin_memory(),
                              gs=torch.empty(self.N, 4).pin_memory())
            # the structs never change between calls: build them once (two ping-pong orientations)
            self._host_args = [(self._state_struct(k), self._state_struct(1 - k), self._io()) for k in (0, 1)]
        h = self._host
        if self._host_ptrs is None or self._host_ptrs[0] is not h:
            self._host_ptrs = (h, _ptr(h['obs']), _ptr(h['reward']), _ptr(h['flags']), _ptr(h['gs']), C.c_void_p(0))
        _, p_obs, p_rew, p_flg, p_gs, p_null = self._host_ptrs
        s_in, s_out, io = self._host_args[self._cur]
        _lib.check(self.lib.rlca_env_step_host(
            self._h, C.byref(s_in), C.byref(s_out), C.byref(io), _ptr(action_host),
            p_obs if want_obs else p_null, p_rew, p_flg, p_gs, self._stream()))
        self._cur = 1 - self._cur
        self._ticked = True
        return h

    def raycast(self, pose, normalise=False, out=None):
        """Stand-alone lidar sweep from arbitrary poses (N,4) -> (N, beams) metres."""
        pose = pose.to(device=self.device, dtype=torch.float32).contiguous()
        out = out if out is not None else torch.empty(self.N, self.beam_mum, device=self.device)
        _lib.check(self.lib.rlca_raycast(self._h, _ptr(pose), _ptr(out), int(normalise), self._stream()))
        return out
