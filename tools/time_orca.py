#!/usr/bin/env python
"""Time one rlca_orca_action launch (the ORCA-DD controller, DESIGN.md §9d) and one rlca_nh_orca_action launch (NH-ORCA,
§9e), map-blind and map-aware (§9f), one rlca_noncoop_action launch with every agent non-cooperative (§9h) and one
rlca_hybrid_action launch with the default thresholds and counting on (§9j), with CUDA events over many launches, on
states after random-action ticks: stage 1 at 171 x 24 agents and the 50-robot circle at 41 x 50.  The six rows
alternate, each timed twice per size.

    python tools/time_orca.py [--launches 2000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rl_collision_avoidance_b200.evaluation import AUTO_RESET  # noqa: E402
from rl_collision_avoidance_b200.evaluation import EpisodeTracker  # noqa: E402
from rl_collision_avoidance_b200.orca import Hybrid, NhOrcaController, NonCooperative, OrcaController  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402


def time_one(scenario, worlds, launches, make, warmup=200):
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=0, auto_reset=AUTO_RESET[scenario])
    env.reset_pose()
    rng = np.random.default_rng(0)
    for _ in range(30):
        a = np.stack([rng.uniform(0, 1, env.N), rng.uniform(-1, 1, env.N)], 1).astype(np.float32)
        env.control_vel(torch.from_numpy(a).cuda())
    ctrl = make(env)
    for _ in range(warmup):
        ctrl()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        ctrl()
    end.record()
    torch.cuda.synchronize()
    us = start.elapsed_time(end) * 1e3 / launches
    fallback = float((ctrl.status() & 1).float().mean())
    st = ctrl.status()
    return {'controller': make.__name__, 'scenario': scenario, 'worlds': worlds, 'agents': env.N, 'us_per_launch': us,
            'fallback_share': fallback, 'status_bit_shares': [float(((st >> b) & 1).float().mean()) for b in range(3)]}


class NonCoop:
    """rlca_noncoop_action (§9h) with every agent masked, overwriting one action buffer."""

    def __init__(self, env):
        self.nc = NonCooperative(env, np.ones(env.N, np.uint8))
        self.action = torch.zeros(env.N, 2, device=env.device)
        self._status = torch.zeros(env.N, dtype=torch.int32, device=env.device)

    def __call__(self):
        return self.nc.apply(self.action)

    def status(self):
        return self._status


class HybridCtl:
    """rlca_hybrid_action (§9j) with the defaults, on a scan stack of three copies of the last scan, counting every
    agent."""

    def __init__(self, env):
        self.hy = Hybrid(env)
        self.stack = env.obs[:, None, :].repeat(1, 3, 1).contiguous()
        self.tracker = EpisodeTracker(env, 1)
        self.action = torch.zeros(env.N, 2, device=env.device)
        self._status = torch.zeros(env.N, dtype=torch.int32, device=env.device)

    def __call__(self):
        return self.hy.apply(self.action, self.stack, self.tracker)

    def status(self):
        return self._status


def OrcaMap(env):
    return OrcaController(env, obstacles=True)


def NhOrcaMap(env):
    return NhOrcaController(env, obstacles=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--launches', type=int, default=2000)
    args = ap.parse_args()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    rows = [time_one(scenario, worlds, args.launches, make) for scenario, worlds in (('stage1', 171), ('circle', 41))
            for _ in range(2) for make in (OrcaController, OrcaMap, NhOrcaController, NhOrcaMap, NonCoop, HybridCtl)]
    print(json.dumps({'card': card, 'power_limit': power, 'launches': args.launches, 'rows': rows}))


if __name__ == '__main__':
    main()
