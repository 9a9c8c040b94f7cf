"""The environment kernels against the oracle on the maps of tests/test_env_maps.py: every path rlca_env_set_map can
pick (small / big map, packed / plain inverse lists, 32- / 64-cell footprint window, aligned / unaligned beams), the
widest small map, rooms smaller than the lidar range, origins off centre and off the grid, open edges.

Per case: ticks of wide random actions, state / scans / local goals / rewards / flags bit-exact against the oracle
every tick; robots teleported onto the last map column and row, the CELL_OOB ring, every pitch-padding column, the
edges, the corners, just past the top and bottom rows and far outside, then observe, a tick and the stand-alone raycast
(raw and normalised) compared; the kernels one tick launches, by name; and counters that the case is not vacuous."""
import ctypes as C
import math
import re

import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, random_actions
from oracle.oracle import OracleWorld, OrcConfig
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario
from test_env_maps import CASE_IDS, MAP_CASES, RANGE_MAX, build_map, oreach, padded

pytestmark = pytest.mark.gpu
PROFILED_TICKS = 3


def _scenario(case, m):
    if case.scenario == 'stage1':
        return make_scenario('stage1', map_=m, robots_per_world=case.K)
    return make_scenario('circle', map_=m, robots_per_world=case.K, radius=case.radius)


def _pair(case, sc, seed):
    """GPU env and oracle of one scenario, auto_reset 1 (as test_evaluation_gpu._pair builds them)."""
    from rl_collision_avoidance_b200.stage_world import StageWorld
    ocfg = fill_config(OrcConfig(), sc, num_worlds=case.worlds, beams=case.beams, auto_reset=1, seed=seed)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    env = StageWorld(case.beams, index=0, scenario=sc, num_worlds=case.worlds, seed=seed, auto_reset=1)
    return env, orc


def _solo(case, sc, n):
    """The oracle with one robot per world: the static part of every scan."""
    ocfg = fill_config(OrcConfig(), sc, num_worlds=n, beams=case.beams)
    ocfg.robots_per_world = 1
    return OracleWorld(ocfg, sc.map.cells, sc.init_tab[:1], sc.goal_tab[:1])


def _kernel_names(env, action):
    """Names of the kernels one tick launches (template arguments included, as torch.profiler reports them)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        env.control_vel(action)
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    norm = lambda s: re.sub(r'\(bool\)1', 'true', re.sub(r'\(bool\)0', 'false', re.sub(r'\(int\)|\s', '', s)))
    return {norm(n) for n in names if 'rlca_' in n}, names


def _expected_kernels(case):
    if case.big:
        return ['rlca_physics_kernel<true>', 'rlca_big_lidar_kernel<3>'], ['rlca_lidar_kernel', 'physics_kernel<false>']
    lidar = f'rlca_lidar_kernel<0,{str(case.beams % 32 == 0).lower()},{str(case.packed).lower()}>'
    return ['rlca_physics_kernel<false>', lidar], ['rlca_big_lidar_kernel', 'physics_kernel<true>']


def _edge_poses(m, rng):
    """(x, y) of robots on the map's edges and beyond them, in world metres: the last column and row, the CELL_OOB
    ring, every pitch-padding column, centres on each edge line, the four corners in and out, the rows just past the
    top and bottom, and far outside."""
    res, W, H, ox, oy = m.resolution, m.grid_w, m.grid_h, m.origin_cx, m.origin_cy
    gw, _ = padded(W, H)
    cx = lambda c: (c - ox + 0.5) * res
    cy = lambda r: (r - oy + 0.5) * res
    xs0, xs1, ys0, ys1 = -ox * res, (W - ox) * res, -oy * res, (H - oy) * res
    pts = []
    for c in [W - 1, W, *range(W + 1, gw - 1), gw - 1, gw, -1, -2, 0]:       # last column, ring, padding, past the pitch
        pts += [(cx(c), cy(H // 2)), (cx(c), cy(int(rng.integers(H)))), (cx(c), cy(H - 1)), (cx(c), cy(0))]
    for r in [H - 1, H, H + 1, -1, -2, 0]:                                     # last row, ring, just past top / bottom
        pts += [(cx(W // 2), cy(r)), (cx(int(rng.integers(W))), cy(r))]
    pts += [(xs0, cy(H // 2)), (xs1, cy(H // 2)), (cx(W // 2), ys0), (cx(W // 2), ys1)]   # straddling each edge
    for c in (0, W - 1, -1, W):                                                # corners, inside and outside
        for r in (0, H - 1, -1, H):
            pts.append((cx(c), cy(r)))
    pts += [(xs1 + 50.0, cy(H // 2)), (xs0 - 40.0, ys0 - 40.0), (cx(W // 2), ys1 + 30.0), (xs1 + 3.0, ys1 + 3.0)]
    return np.asarray(pts, np.float64), (0.5 * (xs0 + xs1), 0.5 * (ys0 + ys1))


class _Coverage:
    """Per-case counters from the oracle's side of the run."""

    def __init__(self, case, sc, n):
        from scipy import ndimage
        self.case, self.m = case, sc.map
        self.solo = _solo(case, sc, n)
        # chessboard distance to the nearest static cell: the footprint window of a robot whose centre cell is within
        # oreach + 1 holds a static cell (the tick reads the template for it)
        self.dt = ndimage.distance_transform_cdt(self.m.cells == 0, metric='chessboard')
        self.c = dict(near_static=0, reverted=0, outside=0, static_hits=0, robot_hits=0, far_static=0)

    def tick(self, orc, scans=False):
        m, c = self.m, self.c
        gx = np.floor(orc.pose[:, 0] * np.float32(1.0 / m.resolution)).astype(np.int64) + m.origin_cx
        gy = np.floor(orc.pose[:, 1] * np.float32(1.0 / m.resolution)).astype(np.int64) + m.origin_cy
        inside = (gx >= 0) & (gx < m.grid_w) & (gy >= 0) & (gy < m.grid_h)
        c['outside'] += int((~inside).sum())
        d = self.dt[np.clip(gy, 0, m.grid_h - 1), np.clip(gx, 0, m.grid_w - 1)]
        c['near_static'] += int((inside & (d <= oreach(m.resolution) + 1)).sum())
        c['reverted'] += int((orc.flags[:, 1] != 0).sum())
        if scans:
            full = orc.raycast(orc.pose)
            alone = self.solo.raycast(orc.pose)
            c['static_hits'] += int(((full == alone) & (alone < RANGE_MAX)).sum())
            c['robot_hits'] += int((full < alone).sum())
            c['far_static'] += int(((full == alone) & (alone < RANGE_MAX) & (alone > RANGE_MAX - 0.2)).sum())


def _compare_tick(env, orc, a, tag):
    env.control_vel(torch.from_numpy(a).cuda())
    orc.step(a)
    assert_state_equal(env, orc, tag)
    assert_outputs_equal(env, orc, tag)
    assert np.array_equal(env.flags.cpu().numpy(), orc.flags), f'{tag}: flags differ'
    assert np.array_equal(env.reward.cpu().numpy().view(np.uint32), orc.reward.view(np.uint32)), f'{tag}: reward'


@pytest.mark.parametrize('case', MAP_CASES, ids=CASE_IDS)
def test_map_case_against_oracle(built, case):
    m = case.map()
    sc = _scenario(case, m)
    env, orc = _pair(case, sc, seed=7)
    N = orc.N
    assert env.cfg.grid_w == case.grid_w and env.cfg.grid_h == case.grid_h
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    assert_state_equal(env, orc, f'{case.name} reset')
    assert_outputs_equal(env, orc, f'{case.name} first observation')
    rng = np.random.default_rng(case.grid_w)

    # the path: kernels of one tick by name; the footprint window from oreach.  The profiler's activity records
    # occasionally lose one kernel of a tick whose launch call it did record, so a tick missing a wanted kernel is
    # profiled again (up to PROFILED_TICKS ticks, each checked against the oracle); a kernel that is not launched is
    # missing from every one of them, and no profiled tick may launch an absent kernel.
    a = random_actions(rng, N, wide=True)
    want, absent = _expected_kernels(case)
    missing = list(want)
    for p in range(PROFILED_TICKS):
        got, raw = _kernel_names(env, torch.from_numpy(a).cuda())
        orc.step(a)
        for k in absent:
            assert not any(k in g for g in got), f'{case.name}: {k} launched; kernels: {sorted(raw)}'
        assert_state_equal(env, orc, f'{case.name} profiled tick {p}')
        assert_outputs_equal(env, orc, f'{case.name} profiled tick {p}')
        missing = [k for k in missing if not any(k in g for g in got)]
        if not missing:
            break
    assert not missing, f'{case.name}: {missing} not launched in {PROFILED_TICKS} ticks; kernels: {sorted(raw)}'
    assert (32 if oreach(case.res) <= 15 else 64) == case.win

    # ticks of wide random actions
    cov = _Coverage(case, sc, N)
    every = 4 if case.kr < 100 else 8
    for t in range(case.ticks):
        _compare_tick(env, orc, random_actions(rng, N, wide=True), f'{case.name} tick {t}')
        cov.tick(orc, scans=t % every == 0)

    # robots 0.6 m inside the edges facing out, driven forwards: off the map where it is open, into the walls elsewhere
    xs0, xs1 = -m.origin_cx * m.resolution, (m.grid_w - m.origin_cx) * m.resolution
    ys0, ys1 = -m.origin_cy * m.resolution, (m.grid_h - m.origin_cy) * m.resolution
    side = rng.integers(4, size=N)
    u = rng.uniform(0.1, 0.9, N)
    pose = np.stack([np.choose(side, [xs0 + 0.6, xs1 - 0.6, xs0 + u * (xs1 - xs0), xs0 + u * (xs1 - xs0)]),
                     np.choose(side, [ys0 + u * (ys1 - ys0), ys0 + u * (ys1 - ys0), ys0 + 0.6, ys1 - 0.6]),
                     np.choose(side, [np.pi, 0.0, -np.pi / 2, np.pi / 2]) + rng.uniform(-0.4, 0.4, N)], 1)
    env.control_pose(torch.from_numpy(pose.astype(np.float32)))
    orc.pose[:] = env.state['pose'].cpu().numpy()
    orc.observe()
    assert_outputs_equal(env, orc, f'{case.name} robots at the edges: observe')
    for t in range(12):
        a = np.stack([rng.uniform(0.8, 1.3, N), rng.uniform(-0.3, 0.3, N)], 1).astype(np.float32)
        _compare_tick(env, orc, a, f'{case.name} drive out, tick {t}')
        cov.tick(orc, scans=t % 3 == 0)
    counts = dict(cov.c)

    # teleports onto and beyond the edges, the ring and the padding columns
    pts, centre = _edge_poses(m, rng)
    reps = -(-len(pts) // N)
    for b in range(reps):
        sel = pts[b * N:(b + 1) * N]
        pose = orc.pose.copy()
        k = len(sel)
        pose[:k, 0:2] = sel
        head = np.arctan2(centre[1] - sel[:, 1], centre[0] - sel[:, 0])        # facing the map ...
        head[1::2] = rng.uniform(-np.pi, np.pi, len(head[1::2]))                 # ... or any heading
        pose[:k, 2] = head
        pose = pose.astype(np.float32)
        tag = f'{case.name} teleport batch {b}'
        for normalise in (False, True):
            got = env.raycast(torch.from_numpy(pose).cuda(), normalise=normalise).cpu().numpy()
            ref = orc.raycast(pose, normalise=normalise)
            bad = np.argwhere(got.view(np.uint32) != ref.view(np.uint32))
            assert len(bad) == 0, f'{tag}: raycast (normalise={normalise}) differs for robots ' \
                f'{np.unique(bad[:, 0])[:8]} at {pose[np.unique(bad[:, 0])[:4], :3].tolist()}'
        env.control_pose(torch.from_numpy(pose[:, :3].copy()))
        orc.pose[:] = env.state['pose'].cpu().numpy()
        orc.observe()
        assert_outputs_equal(env, orc, f'{tag}: observe')
        _compare_tick(env, orc, random_actions(rng, N, wide=True), f'{tag}: tick')

    print(f'{case.name}: {case.worlds} worlds x {case.K} robots x {case.beams} beams, {case.ticks} + 12 ticks, '
          f'{len(pts)} edge poses; ' + ', '.join(f'{k} {v}' for k, v in counts.items()))
    for k in case.need:
        assert counts[k] > 0, f'{case.name}: no {k} in the run ({counts})'
    env.close()


def test_padding_columns_of_stage1(built):
    """Stage 1's own map: robots in the CELL_OOB ring, the padding columns and the first column past the pitch
    (x in [12.2, 15.4) m) see the map as the oracle does: in the stand-alone raycast, from observe and after a tick."""
    from helpers import make_pair
    sc, env, orc = make_pair('stage1', num_worlds=2, seed=3)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    m = sc.map
    gw, _ = padded(m.grid_w, m.grid_h)
    cols = np.arange(m.grid_w, gw)
    pose = orc.pose.copy()
    k = len(cols)
    pose[:k, 0] = (cols - m.origin_cx + 0.5) * m.resolution
    pose[:k, 1] = 0.0
    pose[:k, 2] = np.pi
    pose[k:2 * k, 0] = pose[:k, 0]
    pose[k:2 * k, 1] = np.linspace(-9.0, 9.0, k)
    pose[k:2 * k, 2] = np.linspace(2.0, 4.2, k)
    pose[2 * k, :3] = (13.0, 0.0, np.pi)
    got = env.raycast(torch.from_numpy(pose).cuda()).cpu().numpy()
    ref = orc.raycast(pose)
    assert (ref[2 * k] < RANGE_MAX).sum() == 340
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), \
        f'robots {np.unique(np.argwhere(got != ref)[:, 0])} differ'
    env.control_pose(torch.from_numpy(pose[:, :3].copy()))
    orc.pose[:] = env.state['pose'].cpu().numpy()
    orc.observe()
    assert_outputs_equal(env, orc, 'observe from the padding columns')
    rng = np.random.default_rng(0)
    _compare_tick(env, orc, random_actions(rng, orc.N, wide=True), 'tick from the padding columns')


def test_set_map_rejections(built):
    """Loud errors through rlca_last_error: a resolution whose footprint reaches past 31 cells (oreach 34 at 0.009 m)
    is RLCA_ERR_UNSUPPORTED, a map whose size differs from the config's RLCA_ERR_INVALID."""
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    for res, dw, code, text in ((0.009, 0, 3, b'footprint'), (0.1, 1, 1, b'map size')):
        m = build_map(res, 60, 40, seed=2)
        sc = make_scenario('stage1', map_=m, robots_per_world=4)
        cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=1, beams=512)
        h = C.c_void_p()
        _lib.check(lib.rlca_env_create(C.byref(cfg), C.byref(h)))
        try:
            cells = np.zeros((m.grid_h, m.grid_w + dw), np.uint8)
            rc = lib.rlca_env_set_map(h, cells.ctypes.data_as(C.c_void_p), m.grid_w + dw, m.grid_h)
            assert rc == code, (res, rc, lib.rlca_last_error())
            assert text in lib.rlca_last_error(), lib.rlca_last_error()
        finally:
            lib.rlca_env_destroy(h)
    assert oreach(0.009) == 34 and math.ceil(RANGE_MAX / 0.009) < 2048
