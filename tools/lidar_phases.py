#!/usr/bin/env python
"""Cumulative time of the phases of the small-map lidar launch (rlca_lidar_kernel) on the bench workload (171 stage-1
worlds x 24 robots, 512 beams, the bench's action distribution).

Builds the same -DRLCA_EXPERIMENT copy of librlca.so as tools/physics_phases.py (never over the in-tree library).  With
RLCA_DEBUG >= 20 a tick runs the lidar launch alone: it reads the post-physics state and the outline-cell lists the last
full tick left, and writes only the scans, so replaying it with no physics launch in between times the same work every
time.  For every level 64 such ticks are captured in a CUDA graph and replays are timed with CUDA events; a level's time
is the lidar launch up to that point (plus the gap between two graph nodes):

    20  return at kernel entry
    21  + phase 0: outline-cell list into shared memory, poses of the world's robots
    22  + the first-hit fold (hit[slot] of each viewer = its start cell's first-hit row)
    23  + phase 1: the scatter of the other robots' outline cells (queue + lidar_drain)
    24  the whole lidar launch (+ phase 2, the beam pass)
  none  the whole tick (physics + lidar launch)

Timing experiment only.

    python tools/lidar_phases.py [--tree DIR] [--build-dir DIR] [--rounds 3] [--json OUT]
"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from physics_phases import build_experiment  # noqa: E402

LEVELS = ('20', '21', '22', '23', '24', None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tree', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument('--build-dir', default=None, help='where the experiment library goes (default: a temporary directory)')
    ap.add_argument('--rounds', type=int, default=3, help='sweeps over the levels; the median per level is reported')
    ap.add_argument('--replays', type=int, default=40, help='graph replays (of 64 ticks) timed per level and round')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    tree = os.path.abspath(args.tree)
    build_dir = args.build_dir or tempfile.mkdtemp(prefix='rlca_lidar_phases_')
    lib = build_experiment(tree, build_dir)

    sys.path.insert(0, tree)
    import numpy as np
    import torch
    from rl_collision_avoidance_b200 import _lib
    _lib.LIB_PATH = lib
    from bench import BEAMS, WORLDS_PER_GPU, random_actions
    from rl_collision_avoidance_b200.stage_world import StageWorld

    ticks = 64
    os.environ.pop('RLCA_DEBUG', None)
    env = StageWorld(BEAMS, scenario='stage1', num_worlds=WORLDS_PER_GPU, seed=0, auto_reset=True)
    env.reset_pose()
    rng = np.random.default_rng(1000)
    acts = [torch.from_numpy(random_actions(rng, env.N)).cuda() for _ in range(ticks)]
    ring = torch.empty(ticks, env.N, BEAMS, device='cuda')
    for i in range(200):                        # full ticks: steady-state poses, re-spawns and outline lists
        env.control_vel(acts[i % ticks], obs_out=ring[i % ticks])
    torch.cuda.synchronize()
    # the graphs of the lidar levels never advance the state: everything they replay sees the state left here
    graphs = {}
    for dbg in LEVELS:
        if dbg is None:
            continue
        os.environ['RLCA_DEBUG'] = dbg
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(ticks):
                env.control_vel(acts[i], obs_out=ring[i])
        os.environ.pop('RLCA_DEBUG', None)
        g.replay()
        graphs[dbg] = g
    g = torch.cuda.CUDAGraph()                  # captured last: its replays advance the state
    with torch.cuda.graph(g):
        for i in range(ticks):
            env.control_vel(acts[i], obs_out=ring[i])
    graphs[None] = g
    torch.cuda.synchronize()
    times = {dbg: [] for dbg in LEVELS}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for dbg in LEVELS:
            g = graphs[dbg]
            g.replay()
            e0.record()
            for _ in range(args.replays):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[dbg].append(e0.elapsed_time(e1) / (args.replays * ticks) * 1e3)
    rows = []
    for dbg in LEVELS:
        t = sorted(times[dbg])
        rows.append({'RLCA_DEBUG': dbg, 'us_per_tick': t[len(t) // 2], 'min': t[0], 'max': t[-1]})
    out = {'exp': 'lidar_phases', 'tree': os.path.basename(tree), 'gpu': torch.cuda.get_device_name(), 'rows': rows}
    print(json.dumps(out), flush=True)
    for r in rows:
        print(f"  RLCA_DEBUG={str(r['RLCA_DEBUG']):>4}  {r['us_per_tick']:7.3f} us  [{r['min']:.3f} .. {r['max']:.3f}]",
              flush=True)
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)
    env.close()


if __name__ == '__main__':
    main()
