#!/usr/bin/env python
"""CPU model of the work in the scatter (phase 1) of the small-map lidar launch, per viewer and per CTA, on the bench
workload (stage 1, 24 robots per world, 512 beams, the bench's action distribution), from the oracle, which is bit-exact
with the device.  No GPU.

For every viewer (rlca_lidar_kernel, phase 1a): the outline cells of the other robots of its world (the Cohen edge walk
of each footprint edge, free in-grid cells only, as emit_outline_cells lists them) within lidar range and not behind its
lateral axis; per cell, its inverse list (rlca_walk_tables_host), split into the head a lane drains with its own loads
(6 entries packed, 4 plain) and the rest, a long-list segment.  Work is counted in drain rounds: one round is 32 queued
cells' heads or 32 long-list entries.

  unpooled: a viewer's two warps share its cells and its long-list entries; the CTA waits for its most loaded viewer
  pooled:   the eight warps of the CTA share the work of its four viewers

Prints the distributions and the queue / segment-pool sizes of a CTA at the 99.9th percentile and the maximum, which
set LIDAR_QCAP and LIDAR_PCAP in csrc/rlca_env.cu.  The functions are also the host side of
tests/test_lidar_pool_gpu.py.

    python tools/scatter_work.py [--worlds 171] [--ticks 200] [--every 10] [--json OUT]
"""
import argparse
import ctypes as C
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RPC = 4                      # viewers per CTA (LIDAR_RPC)


def list_lengths(range_cells):
    """Length of the inverse list of every relative cell, (kdim, kdim) indexed [ry, rx], and kr."""
    sys.path.insert(0, ROOT)
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    kr, ns, ne = C.c_int32(), C.c_int32(), C.c_int32()
    _lib.check(lib.rlca_walk_tables_host(C.c_float(range_cells), C.byref(kr), C.byref(ns), C.byref(ne), None, None, None,
                                         None))
    kdim = 2 * kr.value + 1
    keys = np.zeros((ns.value, 2), np.int16)
    keyslot = np.zeros(kdim * kdim, np.uint16)
    off = np.zeros(kdim * kdim + 1, np.uint32)
    ent = np.zeros(max(ne.value, 1), np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_walk_tables_host(C.c_float(range_cells), C.byref(kr), C.byref(ns), C.byref(ne), p(keys),
                                         p(keyslot), p(off), p(ent)))
    return np.diff(off.astype(np.int64)).reshape(kdim, kdim), kr.value, ns.value


def _walk(x0, y0, x1, y1):
    """walk_edge of csrc/rlca_env.cu: the cells of the Cohen walk from (x0, y0), end excluded."""
    dx, dy = x1 - x0, y1 - y0
    sx, sy = (dx > 0) - (dx < 0), (dy > 0) - (dy < 0)
    ax, ay = abs(dx), abs(dy)
    exy = ay - ax
    gx, gy = x0, y0
    for _ in range(ax + ay):
        yield gx, gy
        if exy < 0:
            gx += sx
            exy += 2 * ay
        else:
            gy += sy
            exy -= 2 * ax


def outline_cells(pose, m, half_len, half_wid):
    """Per robot of one world: its outline cells (grid cells in the frame of floor(x * ppm)), free in-grid cells only.
    Corners in float32 without the kernel's FMAs: a corner can land one cell off, which moves a model count by a cell."""
    f = np.float32
    ppm = f(1.0 / m.resolution)
    out = []
    for x, y, th in pose[:, :3]:
        s, c = np.sin(f(th), dtype=f), np.cos(f(th), dtype=f)
        corn = []
        for k in range(4):
            hx = f(half_len) if k in (1, 2) else f(-half_len)
            hy = f(half_wid) if k >= 2 else f(-half_wid)
            corn.append((int(np.floor((hx * c + (-hy * s + f(x))) * ppm)), int(np.floor((hx * s + (hy * c + f(y))) * ppm))))
        cells = []
        for k in range(4):
            for gx, gy in _walk(*corn[k], *corn[(k + 1) & 3]):
                mx, my = gx + m.origin_cx, gy + m.origin_cy
                if 0 <= mx < m.grid_w and 0 <= my < m.grid_h and m.cells[my, mx] == 0:
                    cells.append((gx, gy))
        out.append(np.asarray(cells, np.int64).reshape(-1, 2))
    return out


def viewer_work(pose, m, lens, kr, head, half_len, half_wid, fov):
    """Per robot of one world: (cells queued, cells whose list is longer than the head = segments, long-list entries)."""
    ppm = np.float32(1.0 / m.resolution)
    oc = outline_cells(pose, m, half_len, half_wid)
    halfplane = fov <= 3.1416
    R = len(pose)
    out = np.zeros((R, 3), np.int64)
    for a in range(R):
        x0, y0 = int(np.floor(np.float32(pose[a, 0]) * ppm)), int(np.floor(np.float32(pose[a, 1]) * ppm))
        ct, st = math.cos(pose[a, 2]), math.sin(pose[a, 2])
        cells = [oc[b] for b in range(R) if b != a and len(oc[b])]
        if not cells:
            continue
        q = np.concatenate(cells)
        rx, ry = q[:, 0] - x0, q[:, 1] - y0
        ok = (np.abs(rx) <= kr) & (np.abs(ry) <= kr)
        if halfplane:
            ok &= rx * ct + ry * st >= -3.5
        n = lens[ry[ok] + kr, rx[ok] + kr]
        rest = np.maximum(n - head, 0)
        out[a] = (int(ok.sum()), int((rest > 0).sum()), int(rest.sum()))
    return out


def cta_rows(work):
    """Per CTA of one world (viewers 4k .. 4k + 3): the viewers' (cells, segments, long entries) rows."""
    return [work[k:k + RPC] for k in range(0, len(work), RPC)]


def rounds(rows):
    """Drain rounds of one CTA: (unpooled critical path, pooled)."""
    r = rows[:, 0] / 32.0 + rows[:, 2] / 32.0
    return float(r.max() / 2.0), float(r.sum() / 8.0)


def _dist(x):
    x = np.asarray(x, np.float64)
    return {'mean': float(x.mean()), 'p50': float(np.percentile(x, 50)), 'p99': float(np.percentile(x, 99)),
            'p99.9': float(np.percentile(x, 99.9)), 'max': float(x.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--worlds', type=int, default=171)
    ap.add_argument('--ticks', type=int, default=200)
    ap.add_argument('--every', type=int, default=10, help='ticks between sampled states')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    from bench import BEAMS, random_actions
    from oracle.oracle import OracleWorld, OrcConfig
    from rl_collision_avoidance_b200.scenarios import COMMON, fill_config, make_scenario

    sc = make_scenario('stage1')
    cfg = fill_config(OrcConfig(), sc, num_worlds=args.worlds, beams=BEAMS, auto_reset=True, seed=0)
    orc = OracleWorld(cfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    orc.reset_world()
    orc.reset_pose()
    lens, kr, nslots = list_lengths(cfg.range_cells)
    head = 6 if nslots <= 255 else 4
    R = sc.robots_per_world
    rng = np.random.default_rng(1000)
    acts = [random_actions(rng, orc.N) for _ in range(64)]
    per_viewer, per_cta = [], []
    for t in range(args.ticks):
        orc.step(acts[t % 64])
        if (t + 1) % args.every:
            continue
        for w in range(args.worlds):
            work = viewer_work(orc.pose[w * R:(w + 1) * R].astype(np.float64), sc.map, lens, kr, head,
                               COMMON['half_len'], COMMON['half_wid'], COMMON['fov'])
            per_viewer.append(work)
            per_cta += [(rows.sum(0), *rounds(rows)) for rows in cta_rows(work)]
    v = np.concatenate(per_viewer)
    cta = np.stack([c[0] for c in per_cta])
    unp = np.array([c[1] for c in per_cta])
    pooled = np.array([c[2] for c in per_cta])
    out = {'exp': 'scatter_work', 'worlds': args.worlds, 'ticks': args.ticks, 'every': args.every, 'kr': kr,
           'head_entries': head, 'viewers': len(v), 'ctas': len(cta),
           'viewer_cells': _dist(v[:, 0]), 'viewer_segments': _dist(v[:, 1]), 'viewer_long_entries': _dist(v[:, 2]),
           'cta_cells': _dist(cta[:, 0]), 'cta_segments': _dist(cta[:, 1]), 'cta_long_entries': _dist(cta[:, 2]),
           'rounds_unpooled': _dist(unp), 'rounds_pooled': _dist(pooled)}
    print(json.dumps(out), flush=True)
    f = lambda d: ' '.join(f"{k} {d[k]:7.1f}" for k in ('mean', 'p50', 'p99', 'p99.9', 'max'))
    for k in ('viewer_cells', 'viewer_segments', 'viewer_long_entries', 'cta_cells', 'cta_segments',
              'cta_long_entries', 'rounds_unpooled', 'rounds_pooled'):
        print(f"  {k:20s} {f(out[k])}")
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump(out, fh, indent=1)


if __name__ == '__main__':
    main()
