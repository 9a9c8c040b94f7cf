#!/usr/bin/env python
"""Per-CTA duration of the scatter (phase 1) of the small-map lidar launch against the work its viewers did, on the
bench workload (171 stage-1 worlds x 24 robots, 512 beams, the bench's action distribution).

The launch is one wave (8 CTAs per SM), so it ends when its slowest CTA ends: the early-return levels of
tools/lidar_phases.py measure the maximum over CTAs, this tool the whole distribution.  It builds the same
-DRLCA_EXPERIMENT copy of librlca.so as tools/physics_phases.py (never over the in-tree library), in which
rlca_lidar_kernel records per CTA clock64() at entry, after phase 0 and the first-hit fold, after phase 1 and at the
last warp's exit, the SM it ran on, the cells its viewers queued and the long-list entries (past the head of a list)
they drained.  Every duration is a difference of two clocks of one SM.

The state is replayed as tools/lidar_phases.py does: full ticks to the steady state, then per sample one full tick (the
state advances) and one lidar launch alone over the state it left (RLCA_DEBUG=25: the whole launch, recording; the levels of
tools/lidar_phases.py record nothing), whose CTA records are read.  Samples
of the same state are repeated and the per-CTA median taken, so that a CTA's time is its work, not one draw of the
scheduler.

    python tools/lidar_cta_times.py [--tree DIR] [--build-dir DIR] [--states 16] [--repeats 5] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from physics_phases import build_experiment  # noqa: E402

FIELDS = ('t0', 't1', 't2', 't3', 'sm', 'cells', 'long')


def _stats(x):
    import numpy as np
    x = np.asarray(x, dtype=np.float64)
    return {'mean': float(x.mean()), 'p50': float(np.percentile(x, 50)), 'p99': float(np.percentile(x, 99)),
            'max': float(x.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tree', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument('--build-dir', default=None, help='where the experiment library goes (default: a temporary directory)')
    ap.add_argument('--states', type=int, default=16, help='states sampled (one full tick apart)')
    ap.add_argument('--repeats', type=int, default=5, help='lidar launches per state; the per-CTA median is kept')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    tree = os.path.abspath(args.tree)
    build_dir = args.build_dir or tempfile.mkdtemp(prefix='rlca_lidar_cta_')
    lib = build_experiment(tree, build_dir)

    sys.path.insert(0, tree)
    import numpy as np
    import torch
    from rl_collision_avoidance_b200 import _lib
    _lib.LIB_PATH = lib
    from bench import BEAMS, WORLDS_PER_GPU, random_actions
    from rl_collision_avoidance_b200.stage_world import StageWorld

    env = StageWorld(BEAMS, scenario='stage1', num_worlds=WORLDS_PER_GPU, seed=0, auto_reset=True)
    exp = C.CDLL(lib)
    exp.rlca_exp_cta_read.argtypes = [C.c_void_p, C.c_int]
    ctas = env.num_worlds * ((env.num_env + 3) // 4)
    rec = np.zeros((ctas, len(FIELDS)), dtype=np.uint64)
    os.environ.pop('RLCA_DEBUG', None)
    env.reset_pose()
    rng = np.random.default_rng(1000)
    ticks = 64
    acts = [torch.from_numpy(random_actions(rng, env.N)).cuda() for _ in range(ticks)]
    obs = torch.empty(env.N, BEAMS, device='cuda')
    for i in range(200):                        # full ticks: steady-state poses, re-spawns and outline lists
        env.control_vel(acts[i % ticks], obs_out=obs)
    torch.cuda.synchronize()

    scat, whole, cells, longe, sms = [], [], [], [], []
    for s in range(args.states):
        env.control_vel(acts[s % ticks], obs_out=obs)
        reps = []
        for _ in range(args.repeats + 1):       # the first lidar launch of a state warms its lists into L2
            assert exp.rlca_exp_cta_clear() == 0
            os.environ['RLCA_DEBUG'] = '25'
            env.control_vel(acts[s % ticks], obs_out=obs)
            os.environ.pop('RLCA_DEBUG', None)
            torch.cuda.synchronize()
            assert exp.rlca_exp_cta_read(rec.ctypes.data, ctas) == 0
            reps.append(rec.astype(np.int64).copy())
        reps = np.stack(reps[1:])
        scat.append(np.median(reps[:, :, 2] - reps[:, :, 1], axis=0))
        whole.append(np.median(reps[:, :, 3] - reps[:, :, 0], axis=0))
        cells.append(reps[0, :, 5])
        longe.append(reps[0, :, 6])
        sms.append(reps[0, :, 4])
    scat, whole = np.stack(scat), np.stack(whole)
    cells, longe = np.stack(cells), np.stack(longe)
    # per launch: slowest CTA over the median CTA
    ratio = scat.max(axis=1) / np.median(scat, axis=1)
    # work in drain rounds of the CTA's critical warp is not visible from the device; bin by long-list entries instead
    order = np.argsort(longe.ravel())
    bins = np.array_split(order, 8)
    by_work = [{'long_entries': _stats(longe.ravel()[b]), 'cells': float(cells.ravel()[b].mean()),
                'scatter_cycles': _stats(scat.ravel()[b])} for b in bins]
    props = torch.cuda.get_device_properties(0)
    out = {'exp': 'lidar_cta_times', 'tree': os.path.basename(tree), 'gpu': torch.cuda.get_device_name(),
           'sms': props.multi_processor_count, 'ctas': ctas, 'states': args.states, 'repeats': args.repeats,
           'distinct_sms_used': int(len(np.unique(np.stack(sms)))),
           'scatter_cycles': _stats(scat), 'cta_cycles': _stats(whole),
           'scatter_max_over_p50_per_launch': _stats(ratio),
           'cells_per_cta': _stats(cells), 'long_entries_per_cta': _stats(longe),
           'corr_scatter_long': float(np.corrcoef(scat.ravel(), longe.ravel())[0, 1]),
           'corr_scatter_cells': float(np.corrcoef(scat.ravel(), cells.ravel())[0, 1]),
           'by_long_entries': by_work}
    print(json.dumps(out), flush=True)
    f = lambda d: f"mean {d['mean']:8.0f}  p50 {d['p50']:8.0f}  p99 {d['p99']:8.0f}  max {d['max']:8.0f}"
    print(f"  scatter cycles per CTA      {f(out['scatter_cycles'])}")
    print(f"  whole-CTA cycles            {f(out['cta_cycles'])}")
    print(f"  cells queued per CTA        {f(out['cells_per_cta'])}")
    print(f"  long-list entries per CTA   {f(out['long_entries_per_cta'])}")
    r = out['scatter_max_over_p50_per_launch']
    print(f"  slowest / median CTA scatter per launch: mean {r['mean']:.2f}  max {r['max']:.2f}")
    print(f"  correlation of scatter cycles with long entries {out['corr_scatter_long']:.2f}, with cells "
          f"{out['corr_scatter_cells']:.2f}")
    for b in by_work:
        print(f"    long entries {b['long_entries']['mean']:7.1f} (<= {b['long_entries']['max']:5.0f})  cells "
              f"{b['cells']:6.1f}  scatter cycles {f(b['scatter_cycles'])}")
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump(out, fh, indent=1)
    env.close()


if __name__ == '__main__':
    main()
