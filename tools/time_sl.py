#!/usr/bin/env python
"""Time the SL-policy's device work (DESIGN.md §9g) with CUDA events:
- recording: one rlca_demo_append launch at 171 stage-1 worlds (4104 agent-rows per launch), and the whole recording
  loop of sl.collect (NH-ORCA with the map, env tick and append per tick) in agent-rows/s;
- training: one SL minibatch step at 1024 rows (gather, forward, BC loss, backward, fused Adam), as sl.sl_update runs it.
Each number is taken twice.  Prints one JSON line with the card name and power limit.

    python tools/time_sl.py [--launches 2000] [--steps 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.orca import NhOrcaController  # noqa: E402
from rl_collision_avoidance_b200.sl import DemoSet, collect, sl_update  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402

WORLDS = 171


def events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def time_append(env, launches, warmup=100, ticks=50):
    """µs per rlca_demo_append launch.  The dataset holds `ticks` ticks and its count is zeroed every `ticks` launches
    (one small memset), so every timed launch copies its rows."""
    demo = DemoSet(env, env.N * ticks)
    stack = torch.rand(env.N, 3, 512, device='cuda')
    action = torch.rand(env.N, 2, device='cuda')
    for i in range(warmup):
        if i % ticks == 0:
            demo.counter.zero_()
        demo.append(action, stack)
    start, end = events()
    start.record()
    for i in range(launches):
        if i % ticks == 0:
            demo.counter.zero_()
        demo.append(action, stack)
    end.record()
    torch.cuda.synchronize()
    assert demo.count() == env.N * ((launches - 1) % ticks + 1)
    us = start.elapsed_time(end) * 1e3 / launches
    row_bytes = (3 * 512 + 4 + 2) * 4
    return {'us_per_launch': us, 'agent_rows_per_s': env.N / us * 1e6,
            'write_GB_per_s': env.N * row_bytes / us * 1e-3}


def time_collect(env, rows):
    ctrl = NhOrcaController(env, obstacles=True)
    collect(env, ctrl, env.N * 20)                      # warm-up: every launch shape of the loop
    start, end = events()
    start.record()
    data = collect(env, ctrl, rows)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end)
    return {'rows': int(data[0].shape[0]), 'ms': ms, 'agent_rows_per_s': data[0].shape[0] / ms * 1e3}


def time_step(steps, batch=1024, warmup=20):
    n = batch * 64
    data = (torch.rand(n, 1536, device='cuda') - 0.5, torch.randn(n, 4, device='cuda'), torch.rand(n, 2, device='cuda'))
    pol = CNNPolicy(frames=3, action_space=2, seed=0, max_batch=batch)
    opt = Adam(pol.parameters(), lr=1e-4)
    g = torch.Generator(device='cuda')
    g.manual_seed(0)
    sl_update(pol, opt, data, batch, max(1, warmup // 64), generator=g)
    epochs = max(1, steps // 64)
    start, end = events()
    start.record()
    sl_update(pol, opt, data, batch, epochs, generator=g)
    end.record()
    torch.cuda.synchronize()
    return {'batch': batch, 'steps': epochs * 64, 'ms_per_step': start.elapsed_time(end) / (epochs * 64)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--launches', type=int, default=2000)
    ap.add_argument('--steps', type=int, default=256)
    ap.add_argument('--collect-rows', type=int, default=400000)
    args = ap.parse_args()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    env = StageWorld(512, scenario='stage1', num_worlds=WORLDS, seed=0, auto_reset=1)
    out = {'card': card, 'power_limit': power, 'agents': env.N,
           'append': [time_append(env, args.launches) for _ in range(2)],
           'collect': [time_collect(env, args.collect_rows) for _ in range(2)],
           'sl_step': [time_step(args.steps) for _ in range(2)]}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
