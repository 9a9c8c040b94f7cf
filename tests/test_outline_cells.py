"""The small-map physics launch keeps the footprint outline cells of a world in a shared array (outline_mark in
csrc/rlca_env.cu): edge e owns the slots e * ec .. e * ec + ec - 1, ec = 2 (ceil(longest side * ppm) + 1), filled with
walk_edge's cells in order and OC_NONE after them; the test, the windows and the outline-cell list for the lidar all
read that array, and robots that keep their pose reuse it for the list.

CPU: the slots of every edge of real footprints, at the shipped resolutions, hold the whole walk (no cell is dropped).
GPU: the outline-cell list the physics launch leaves for the lidar (reused entries of robots that kept their pose,
re-walked edges of reverted and re-spawned robots) yields the same scans as a stand-alone sweep from the final poses,
which builds its list from those poses alone, in crowded worlds with robots against the walls."""
import math

import numpy as np
import pytest

HALF_LEN, HALF_WID = 0.22, 0.19          # scenarios.COMMON
RESOLUTIONS = (0.2, 0.01)                 # stage 1 / stage 2, circle.world
OC_UNROLL = 4


def walk_edge(x0, y0, x1, y1):
    """csrc/rlca_env.cu walk_edge, step for step."""
    dx, dy = x1 - x0, y1 - y0
    sx, sy = (dx > 0) - (dx < 0), (dy > 0) - (dy < 0)
    ax, ay = abs(dx), abs(dy)
    bx, by = 2 * ax, 2 * ay
    exy = ay - ax
    out = []
    gx, gy = x0, y0
    for _ in range(ax + ay):
        out.append((gx, gy))
        if exy < 0:
            gx += sx
            exy += by
        else:
            gy += sy
            exy -= bx
    return out


def edge_slots(x0, y0, x1, y1, ec):
    """outline_mark's slots of one edge: the walk OC_UNROLL cells per chunk while cells remain, stores below ec, then
    OC_NONE (None here) up to ec."""
    cells = walk_edge(x0, y0, x1, y1)
    slots = [None] * ec
    s0 = 0
    while s0 < len(cells):
        for u in range(OC_UNROLL):
            if s0 + u < ec:
                slots[s0 + u] = cells[s0 + u] if s0 + u < len(cells) else None
        s0 += OC_UNROLL
    return slots


def oreach(res):
    return math.ceil(math.hypot(HALF_LEN, HALF_WID) / res) + 1


def edge_cap(res):
    return 2 * (math.ceil(2 * max(HALF_LEN, HALF_WID) / res) + 1)


def _corners(x, y, th, ppm):
    """corner_cell in float32 (fmaf-free restatement: the offsets stay within a cell of the kernel's)."""
    f = np.float32
    s, c = np.sin(f(th), dtype=f), np.cos(f(th), dtype=f)
    out = []
    for k in range(4):
        hx = f(HALF_LEN) if k in (1, 2) else f(-HALF_LEN)
        hy = f(HALF_WID) if k >= 2 else f(-HALF_WID)
        px = hx * c + (-hy * s + f(x))
        py = hx * s + (hy * c + f(y))
        out.append((int(np.floor(px * f(ppm))), int(np.floor(py * f(ppm)))))
    return out


@pytest.mark.parametrize('res', RESOLUTIONS)
def test_edge_slots_hold_the_whole_walk(res):
    rng = np.random.default_rng(7)
    ppm = 1.0 / res
    ec = edge_cap(res)
    longest = 0
    for _ in range(400 if res < 0.1 else 4000):
        corn = _corners(rng.uniform(-30, 30), rng.uniform(-30, 30), rng.uniform(-math.pi, math.pi), ppm)
        for k in range(4):
            (x0, y0), (x1, y1) = corn[k], corn[(k + 1) & 3]
            ref = walk_edge(x0, y0, x1, y1)
            assert len(ref) <= ec
            assert edge_slots(x0, y0, x1, y1, ec) == ref + [None] * (ec - len(ref))
            longest = max(longest, len(ref))
    assert longest >= ec // 2


# ------------------------------------------------------------------------------------------------------------- GPU
def _crowd(env, sc, rng, worlds):
    """Press the robots of the first `worlds` worlds against each other (pairs 0.3 m apart, closer than a footprint) and
    against the walls (centres 2-3 cells from a non-free cell)."""
    import torch
    from scipy import ndimage
    m = sc.map
    cells = np.asarray(m.cells)
    dt = ndimage.distance_transform_cdt(cells == 0, metric='chessboard')
    rows, cols = np.nonzero((dt >= 2) & (dt <= 3))
    R = sc.robots_per_world
    pose = env.state['pose'].cpu().numpy()
    for w in range(worlds):
        for r in range(R):
            a = w * R + r
            if r % 3 == 0:               # against a wall
                k = rng.integers(len(rows))
                pose[a, 0] = (cols[k] - m.origin_cx + 0.5) * m.resolution
                pose[a, 1] = (rows[k] - m.origin_cy + 0.5) * m.resolution
            elif r % 3 == 1:             # next to the previous robot
                pose[a, 0] = pose[a - 1, 0] + 0.3
                pose[a, 1] = pose[a - 1, 1] + rng.uniform(-0.1, 0.1)
            pose[a, 2] = rng.uniform(-math.pi, math.pi)
    env.state['pose'].copy_(torch.from_numpy(pose))
    return dt


def _not_allfree(env, sc, dt):
    """Robots whose footprint reaches a non-free cell (the kernel reads the template for them)."""
    m = sc.map
    pose = env.state['pose'].cpu().numpy()
    cx = np.floor(pose[:, 0] / m.resolution).astype(int) + m.origin_cx
    cy = np.floor(pose[:, 1] / m.resolution).astype(int) + m.origin_cy
    inside = (cx >= 0) & (cx < dt.shape[1]) & (cy >= 0) & (cy < dt.shape[0])
    d = dt[np.clip(cy, 0, dt.shape[0] - 1), np.clip(cx, 0, dt.shape[1] - 1)]
    return int((~inside | (d <= oreach(m.resolution) + 1)).sum())


@pytest.mark.gpu
@pytest.mark.parametrize('scenario,R,auto_reset', [('stage1', 1, 1), ('stage1', 24, 1), ('stage1', 24, 0),
                                                   ('stage1', 44, 1), ('stage1', 64, 1), ('stage2', None, 2)])
def test_tick_list_gives_the_scans_of_the_final_poses(built, scenario, R, auto_reset):
    import torch
    from helpers import make_pair, random_actions
    worlds = 6
    sc, env, _ = make_pair(scenario, num_worlds=worlds, auto_reset=auto_reset, seed=3, robots_per_world=R, gpu=True)
    env.reset_pose()
    rng = np.random.default_rng(3)
    dt = _crowd(env, sc, rng, worlds // 2)
    reverted = respawned = near_wall = 0
    for t in range(40):
        near_wall += _not_allfree(env, sc, dt)
        env.control_vel(torch.from_numpy(random_actions(rng, env.N, wide=True)).cuda())
        obs = env.obs.cpu().numpy()
        ref = env.raycast(env.state['pose'], normalise=True).cpu().numpy()
        bad = np.argwhere(obs.view(np.uint32) != ref.view(np.uint32))
        assert len(bad) == 0, f'{scenario} R={R} tick {t}: agents {np.unique(bad[:, 0])[:8]}'
        flags = env.flags.cpu().numpy()
        reverted += int(((flags[:, 1] != 0) & (flags[:, 3] == 0)).sum())
        respawned += int((flags[:, 3] != 0).sum())
    print(f'{scenario} R={R} auto_reset={auto_reset}: reverted {reverted}, re-spawned {respawned}, '
          f'robot-ticks near a wall {near_wall}')
    assert near_wall > 0
    if auto_reset != 1:
        assert reverted > 0
    if auto_reset == 1 and R != 1:
        assert respawned > 0
    env.close()
