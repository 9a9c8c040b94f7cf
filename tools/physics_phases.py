#!/usr/bin/env python
"""Cumulative time of the phases of the physics launch on the bench workload (171 stage-1 worlds x 24 robots, 512
beams, the bench's action distribution).

Builds an -DRLCA_EXPERIMENT copy of librlca.so into its own directory (never over the in-tree library): rlca_env.cu of
the tree is compiled with the early returns enabled and linked with the tree's other objects (run build() first).
For every RLCA_DEBUG level it captures 64 ticks in a CUDA graph and times replays of it with CUDA events.  With
RLCA_DEBUG set the experiment library runs the physics launch alone, so a level's time is the physics launch up to
that point (plus the gap between two graph nodes):

     6  return at kernel entry               3  + phase A (state loads, integration)
     4  + windows_mark                       5  + windows_test (collision test)
     8  + phase B (revert, reward / done)    9  + re-spawn
    10  + rebuild and state / output stores 11  the whole physics launch (+ outline-cell list)
  none  the whole tick (physics + lidar launch)

With an early return the state is not advanced; the warm-up runs full ticks so that the inputs are those of the
workload in steady state.  Timing experiment only.

    python tools/physics_phases.py [--tree DIR] [--build-dir DIR] [--rounds 3] [--json OUT]
"""
import argparse
import glob
import json
import os
import subprocess
import sys
import tempfile

LEVELS = ('6', '3', '4', '5', '8', '9', '10', '11', None)


def build_experiment(tree, out_dir):
    csrc = os.path.join(tree, 'rl_collision_avoidance_b200', 'csrc')
    objs = [o for o in sorted(glob.glob(os.path.join(tree, 'rl_collision_avoidance_b200', 'build', '*.o')))
            if os.path.basename(o) != 'rlca_env.o']
    if not objs:
        raise SystemExit('no objects under rl_collision_avoidance_b200/build: run __graft_entry__.build() first')
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    arch = ['-gencode', 'arch=compute_90a,code=sm_90a']
    os.makedirs(out_dir, exist_ok=True)
    obj = os.path.join(out_dir, 'rlca_env_exp.o')
    lib = os.path.join(out_dir, 'librlca_exp.so')
    subprocess.check_call([nvcc] + arch + ['-O3', '-std=c++17', '-Xcompiler', '-fPIC', '-fmad=false', '-DRLCA_EXPERIMENT',
                                           '-I', os.path.join(tree, 'include'), '-c', os.path.join(csrc, 'rlca_env.cu'),
                                           '-o', obj])
    subprocess.check_call([nvcc] + arch + ['-shared', '-o', lib, obj] + objs)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tree', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument('--build-dir', default=None, help='where the experiment library goes (default: a temporary directory)')
    ap.add_argument('--rounds', type=int, default=3, help='sweeps over the levels; the median per level is reported')
    ap.add_argument('--replays', type=int, default=40, help='graph replays (of 64 ticks) timed per level and round')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    tree = os.path.abspath(args.tree)
    build_dir = args.build_dir or tempfile.mkdtemp(prefix='rlca_phases_')
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
    graphs = {}
    for dbg in LEVELS:
        if dbg is None:
            os.environ.pop('RLCA_DEBUG', None)
        else:
            os.environ['RLCA_DEBUG'] = dbg
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(ticks):
                env.control_vel(acts[i], obs_out=ring[i])
        os.environ.pop('RLCA_DEBUG', None)
        g.replay()
        graphs[dbg] = g
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
    out = {'exp': 'physics_phases', 'tree': os.path.basename(tree), 'gpu': torch.cuda.get_device_name(), 'rows': rows}
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
