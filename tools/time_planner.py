#!/usr/bin/env python
"""Cost of the global planner (DESIGN.md §9w), CUDA events round many calls, two passes, on the card named in the
output (with its power limit and maximum SM clock):
  - rlca_plan_fields with every row re-planned (the cache cleared before each call, outside the events) and with no
    row re-planned, and rlca_plan_waypoints, at stage 1 171 x 24, stage 2 24 x 44 and arenas 1024 x 16;
  - an evaluation of `stage2.pth` with and without --planner on arenas (1024 x 16), per tick (the whole evaluate() call
    over its ticks, set-up included).

    python tools/time_planner.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.planner import Planner  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402

STAGE2 = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')


def events(fn, n, before=None):
    """Mean ms of fn() over n calls, CUDA events round each call (`before` runs outside the events)."""
    total = 0.0
    for _ in range(n):
        if before is not None:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1)
    return total / n


def scenario(name, K=16):
    return make_scenario('arena', robots_per_world=K, arenas=64) if name == 'arena' else make_scenario(name)


def launches():
    for name, W in (('stage1', 171), ('stage2', 24), ('arena', 1024)):
        sc = scenario(name)
        env = StageWorld(512, scenario=sc, num_worlds=W, seed=0, auto_reset=AUTO_RESET[name])
        env.reset_world()
        env.reset_pose()
        if sc.layout is not None:
            env.random_layout()
        p = Planner(env)
        p.update()
        lib, cfg, st = env.lib, env.cfg, env._state_struct(env._cur)
        import ctypes as C
        fields = lambda: lib.rlca_plan_fields(C.byref(cfg), C.byref(p._t), C.byref(p._st), C.byref(st), env._stream())
        wp = lambda: lib.rlca_plan_waypoints(C.byref(cfg), C.byref(p._t), C.byref(p._st), C.byref(st),
                                             C.c_void_p(env.gs.data_ptr()), C.c_void_p(p.gs.data_ptr()),
                                             env._stream())
        clear = lambda: p.entry.fill_(-1)
        for pas in range(2):
            n_all = 3 if name == 'stage2' else 10
            t_all = events(fields, n_all, clear)
            t_none = events(fields, 200)
            t_wp = events(wp, 200)
            print('%s %d x %d pass %d: fields all re-planned %.3f ms  none re-planned %.1f us  waypoints %.1f us  '
                  '(largest field %d cells)' % (name, W, sc.robots_per_world, pas, t_all, 1e3 * t_none, 1e3 * t_wp,
                                                p.tables.max_area), flush=True)
        del p, env
        torch.cuda.empty_cache()


def ticks():
    sc = scenario('arena', 16)
    for pas in range(2):
        for steer in (None, True):
            env = StageWorld(512, scenario=sc, num_worlds=1024, seed=0)
            pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
            pol.load_state_dict(torch.load(STAGE2, map_location='cuda'))
            planner = Planner(env, steer) if steer is not None else None
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            out = evaluate(env, pol, 1, 300, check_every=1000, planner=planner)
            e1.record()
            e1.synchronize()
            print('evaluation arena 1024 x 16, %d ticks, pass %d, %s: %.3f ms per tick'
                  % (out['ticks'], pas, 'with --planner' if steer else 'without planner',
                     e0.elapsed_time(e1) / out['ticks']), flush=True)
            del env, pol, planner
            torch.cuda.empty_cache()


def main():
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info), flush=True)
    launches()
    ticks()


if __name__ == '__main__':
    main()
