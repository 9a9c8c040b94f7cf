#!/usr/bin/env python
"""The raster gap of the map-aware ORCA baselines (DESIGN.md §9f), on the CPU: how often the simulator's collision
rule blocks a pose whose centre is at least r_o from every obstacle segment.

The obstacle lines keep a robot's centre r_o clear of the boundary segments, but the physics blocks a robot when a
static cell lies on its rasterised outline (robot_outline / grid_blocks of the oracle, oracle/sim_oracle.c), and that
cell can lie up to about one cell beyond the geometric footprint.  For uniformly random poses (x, y, heading) on a
map, the centre's float64 distance to the nearest boundary segment is measured, and each pose with a free centre cell
and a distance >= r_o is tested by the oracle: one robot per world, placed at the pose and given the command
(v, w) = (0, 1e-30), which moves it (so that its outline is tested) while leaving the pose unchanged.  The pose is
blocked when the tick reports a crash.

    python tools/orca_raster_gap.py [--samples 100000] [--r-o 0.35 0.45 0.55]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.oracle import OracleWorld, OrcConfig  # noqa: E402
from rl_collision_avoidance_b200 import _lib  # noqa: E402
from rl_collision_avoidance_b200.orca import ObstacleSet  # noqa: E402
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario  # noqa: E402

CHUNK = 20000


def segment_distance(points, x, y):
    """Least float64 distance from each (x, y) to the segments (S, 4)."""
    a = points[:, 0:2].astype(np.float64)
    e = points[:, 2:4].astype(np.float64) - a
    best = np.full(len(x), np.inf)
    for k in range(0, len(a), 64):
        A, E = a[k:k + 64], e[k:k + 64]
        rx, ry = x[:, None] - A[None, :, 0], y[:, None] - A[None, :, 1]
        t = np.clip((rx * E[:, 0] + ry * E[:, 1]) / (E ** 2).sum(1), 0.0, 1.0)
        best = np.minimum(best, np.hypot(rx - t * E[:, 0], ry - t * E[:, 1]).min(1))
    return best


def blocked(m, x, y, th):
    """The oracle's verdict for each pose: True when the tick with (0, 1e-30) reports a crash."""
    out = np.zeros(len(x), bool)
    sc = make_scenario('stage1', map_=m, robots_per_world=1)
    for s in range(0, len(x), CHUNK):
        n = min(CHUNK, len(x) - s)
        cfg = fill_config(OrcConfig(), sc, num_worlds=n, beams=8, auto_reset=0)
        orc = OracleWorld(cfg, m.cells, sc.init_tab, sc.goal_tab)
        orc.pose[:, 0], orc.pose[:, 1], orc.pose[:, 2] = x[s:s + n], y[s:s + n], th[s:s + n]
        orc.goal[:, 0:2] = 1e4                                   # never reached
        action = np.zeros((n, 2), np.float32)
        action[:, 1] = 1e-30
        orc.step(action)
        assert np.array_equal(orc.pose[:, 2], th[s:s + n].astype(np.float32))
        out[s:s + n] = orc.flags[:, 1] != 0
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--samples', type=int, default=100000)
    ap.add_argument('--r-o', type=float, nargs='+', default=[0.35, 0.45, 0.55])
    ap.add_argument('--seed', type=int, default=0)
    args = ap.parse_args()
    rows = []
    for name in ('stage1', 'stage2'):
        m = make_scenario(name).map
        cfg = fill_config(_lib.EnvConfig(), make_scenario(name), num_worlds=1, beams=512)
        pts, _, _ = ObstacleSet(cfg, m.cells, 1.35).segments()
        rng = np.random.default_rng(args.seed)
        x0, y0 = -m.origin_cx * m.resolution, -m.origin_cy * m.resolution
        x = rng.uniform(x0, x0 + m.grid_w * m.resolution, args.samples).astype(np.float32)
        y = rng.uniform(y0, y0 + m.grid_h * m.resolution, args.samples).astype(np.float32)
        th = rng.uniform(-np.pi, np.pi, args.samples).astype(np.float32)
        ci = np.floor(x.astype(np.float64) / m.resolution).astype(int) + m.origin_cx
        cj = np.floor(y.astype(np.float64) / m.resolution).astype(int) + m.origin_cy
        free = m.cells[np.clip(cj, 0, m.grid_h - 1), np.clip(ci, 0, m.grid_w - 1)] == 0
        dist = segment_distance(pts, x.astype(np.float64), y.astype(np.float64))
        hit = blocked(m, x[free], y[free], th[free])
        d = dist[free]
        for r_o in args.r_o:
            sel = d >= r_o
            rows.append({'map': name, 'r_o': r_o, 'poses': int(sel.sum()), 'blocked': int(hit[sel].sum()),
                         'share': float(hit[sel].mean()) if sel.any() else float('nan'),
                         'largest_blocked_clearance': float(d[sel & hit].max()) if (sel & hit).any() else None})
        for lo, hi in ((0.0, 0.1), (0.1, 0.2), (0.2, 0.25), (0.25, 0.29), (0.29, 0.31), (0.31, 0.35)):
            sel = (d >= lo) & (d < hi)
            rows.append({'map': name, 'clearance': [lo, hi], 'poses': int(sel.sum()), 'blocked': int(hit[sel].sum())})
    print(json.dumps({'samples_per_map': args.samples, 'seed': args.seed, 'rows': rows}))


if __name__ == '__main__':
    main()
