#!/usr/bin/env python
"""The cost numbers of DESIGN.md §9v, each timed with CUDA events round every call, in two alternating passes:
  - the layout kernels at 1024 worlds x 16 robots: rlca_layout_arena (pick 0 and 1) and rlca_layout_arena_respawn with
    every world re-laid, against rlca_layout_random and rlca_layout_respawn at the same shape;
  - one tick (rlca_env_step) on the arena map (64 arenas of 10 m) at 171 x 16 and 1024 x 16, against the random
    scenario's tick on circle.world at the same shapes, zero actions from a fresh layout;
  - the map set-up: StageWorld construction (rlca_env_set_map with its first-hit table build, and the upload of the
    arena tables) on the arena map and on circle.world, host clock round a synchronised call.
Prints the card, power limit and maximum SM clock first.

    python tools/time_arena.py
"""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200 import _lib  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402

K, CALLS = 16, 200


def _per_call_us(fn, before=None, calls=CALLS):
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(calls)]
    for _ in range(10):
        if before:
            before()
        fn()
    for e0, e1 in evs:
        if before:
            before()
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return 1e3 * float(np.mean([e0.elapsed_time(e1) for e0, e1 in evs]))


def _env(sc, worlds):
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=0, auto_reset=0)
    env.reset_world()
    env.random_layout()
    return env


def layout_times(arena, rnd):
    """(name, us) of the layout launches on envs `arena` and `rnd`."""
    out = []
    status = torch.empty(arena.num_worlds, dtype=torch.int32, device='cuda')
    for name, env in (('arena', arena), ('random', rnd)):
        lay = env.sc.layout
        params = _lib.LayoutParams(lay.side, lay.separation, lay.min_travel)
        st = env._state_struct(env._cur)
        sp = C.c_void_p(status.data_ptr())
        if name == 'arena':
            for pick in (0, 1):
                fn = lambda p=pick: _lib.check(env.lib.rlca_layout_arena(C.byref(env.cfg), C.byref(params),
                                                                         C.byref(env._arena), p, C.byref(st), sp,
                                                                         env._stream()))
                out.append(('rlca_layout_arena pick %d' % pick, _per_call_us(fn)))
            resp = lambda: _lib.check(env.lib.rlca_layout_arena_respawn(
                C.byref(env.cfg), C.byref(params), C.byref(env._arena), 1, C.byref(st), C.c_void_p(env.flags.data_ptr()),
                C.c_void_p(env.live.data_ptr()), sp, env._stream()))
            rname = 'rlca_layout_arena_respawn, every world re-laid'
        else:
            fn = lambda: _lib.check(env.lib.rlca_layout_random(C.byref(env.cfg), C.byref(params), C.byref(st), sp,
                                                               env._stream()))
            out.append(('rlca_layout_random', _per_call_us(fn)))
            resp = lambda: _lib.check(env.lib.rlca_layout_respawn(
                C.byref(env.cfg), C.byref(params), C.byref(st), C.c_void_p(env.flags.data_ptr()),
                C.c_void_p(env.live.data_ptr()), sp, env._stream()))
            rname = 'rlca_layout_respawn, every world re-laid'
        latch = lambda e=env: e.state['meta'][:, 3].fill_(1)
        out.append((rname, _per_call_us(resp, before=latch)))
        torch.cuda.synchronize()
        out.append(('worlds the last re-layout could not fill', int(status.count_nonzero())))
        env.state['meta'][:, 3].zero_()
        env.live.fill_(1)
    return out


def tick_us(env):
    action = torch.zeros(env.N, 2, device='cuda')
    stacks = torch.empty(2, env.N, 3, 512, device='cuda')
    stacks[0] = env.obs[:, None, :]
    return _per_call_us(lambda: env.control_vel(action, live=env.live, stack_in=stacks[0], stack_out=stacks[1]))


def setup_s(sc, worlds=16):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=0, auto_reset=0)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    del env
    return dt


def main():
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info))
    arena_sc = make_scenario('arena', robots_per_world=K)
    random_sc = make_scenario('random', robots_per_world=K)
    fh = ((arena_sc.map.grid_w + 2 + 15) // 16 * 16 - 2) * arena_sc.map.grid_h * 256
    print('arena map: %d x %d cells at %g m, first-hit table %.1f MB; %d arenas, %d placeable cells'
          % (arena_sc.map.grid_w, arena_sc.map.grid_h, arena_sc.map.resolution, fh / 2 ** 20,
             arena_sc.layout.count, len(arena_sc.layout.tables.cells)), flush=True)
    for p in range(2):
        for name, sc in (('arena', arena_sc), ('circle.world (random)', random_sc)):
            setup_s(sc)                                              # warm: module load, first allocation
            print('pass %d: set-up of a 16-world env on %s: %.1f ms' % (p + 1, name, 1e3 * setup_s(sc)), flush=True)
    arena, rnd = _env(arena_sc, 1024), _env(random_sc, 1024)
    for p in range(2):
        for name, us in layout_times(arena, rnd):
            if isinstance(us, int):
                print('pass %d: 1024 x %d: %s: %d' % (p + 1, K, name, us), flush=True)
            else:
                print('pass %d: 1024 x %d: %s %.1f us (mean of %d calls)' % (p + 1, K, name, us, CALLS), flush=True)
    del arena, rnd
    torch.cuda.empty_cache()
    for worlds in (171, 1024):
        envs = (('arena map', _env(arena_sc, worlds)), ('circle.world (random)', _env(random_sc, worlds)))
        for p in range(2):
            for name, env in envs:
                print('pass %d: %d x %d: one tick on %s %.1f us (mean of %d calls)'
                      % (p + 1, worlds, K, name, tick_us(env), CALLS), flush=True)
        del envs
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
