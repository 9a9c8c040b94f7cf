#!/usr/bin/env python
"""The random-scenario results of DESIGN.md §9i: evaluate.py --scenario random for K in {4, 8, 16, 32} robots on the
default 10 m square, 1024 worlds, seed 0, one episode per robot, for stage2.pth, stage1_2.pth, NH-ORCA+map and ORCA-DD.
Prints the card and power limit, one markdown row per run with the number of distinct layouts among its worlds, and the
time of one rlca_layout_random launch at 4096 x 8 and 4096 x 64 agents (CUDA events over many launches).

    python tools/random_table.py
"""
import contextlib
import ctypes as C
import io
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import evaluate  # noqa: E402
from rl_collision_avoidance_b200 import _lib  # noqa: E402
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario, random_layout_host  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
CONTROLLERS = [('`stage2.pth`', ['--policy', os.path.join(CKPT, 'stage2.pth')]),
               ('`stage1_2.pth`', ['--policy', os.path.join(CKPT, 'stage1_2.pth')]),
               ('NH-ORCA+map', ['--baseline', 'nh-orca', '--orca-map']),
               ('ORCA-DD', ['--baseline', 'orca'])]
WORLDS, SEED = 1024, 0


def distinct_worlds(K, worlds, seed):
    """Distinct (start, goal, heading) layouts among the worlds, from the host twin of the device sampler."""
    sc = make_scenario('random', robots_per_world=K)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=worlds, beams=512, seed=seed)
    z = np.zeros((K * worlds, 4), np.float32)
    pose, goal, _, status = random_layout_host(cfg, sc.layout, z, z, z)
    assert not status.any()
    rows = np.concatenate((pose[:, 0:3], goal[:, 0:2]), 1).reshape(worlds, -1)
    return len(np.unique(rows, axis=0))


def row(name, K, ticks, distinct, m):
    f = lambda key: '–' if m[key][0] != m[key][0] else '%.3f ± %.3f' % m[key]
    return '| %s | %d | %d | %d | %d | %d | %.3f | %.3f | %.3f | %d | %s | %s | %s |' % (
        name, K, WORLDS, distinct, ticks, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
        m['unfinished'], f('extra_time'), f('extra_distance'), f('average_speed'))


def time_layout(K, side, worlds=4096, launches=200):
    """Mean time of one rlca_layout_random launch, CUDA events round `launches` back-to-back launches."""
    from rl_collision_avoidance_b200.stage_world import StageWorld
    sc = make_scenario('random', robots_per_world=K, side=side)
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=SEED, auto_reset=0)
    env.reset_world()
    env.reset_pose()
    params = _lib.LayoutParams(sc.layout.side, sc.layout.separation, sc.layout.min_travel)
    st = env._state_struct(env._cur)
    status = torch.empty(worlds, dtype=torch.int32, device=env.device)
    stream = env._stream()
    launch = lambda: _lib.check(env.lib.rlca_layout_random(C.byref(env.cfg), C.byref(params), C.byref(st),
                                                           C.c_void_p(status.data_ptr()), stream))
    for _ in range(10):
        launch()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(launches):
        launch()
    t1.record()
    torch.cuda.synchronize()
    assert not status.any()
    return t0.elapsed_time(t1) * 1e3 / launches


def main():
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    for K, side in ((8, 10.0), (64, 20.0)):
        print('rlca_layout_random, 4096 worlds x %d robots (%g m square): %.1f us per launch (mean of 200)'
              % (K, side, time_layout(K, side)), flush=True)
    print('| controller | K | worlds | distinct worlds | ticks | episodes | success | crash | time-out | unfinished | '
          'extra time | extra distance | average speed |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|---|')
    for K in (4, 8, 16, 32):
        distinct = distinct_worlds(K, WORLDS, SEED)
        for name, who in CONTROLLERS:
            with contextlib.redirect_stdout(io.StringIO()):
                out = evaluate.main(['--scenario', 'random', '--random-robots', str(K), '--num-worlds', str(WORLDS),
                                     '--seed', str(SEED)] + who)
            print(row(name, K, out['ticks'], distinct, out['metrics']), flush=True)
            del out
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
