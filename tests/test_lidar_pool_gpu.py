"""The small-map lidar's pooled scatter (rlca_lidar_kernel, phase 1) against the oracle on crowded worlds: every robot of
a world packed round the first one, so that a CTA's viewers queue more cells than the CTA's queue holds and more long
lists than its segment pool holds, and the in-place drains behind both capacities run.  The host model of
tools/scatter_work.py shows that each case's state is past the capacities; then observe, the stand-alone raycast (raw
and normalised) and ticks are compared bit for bit, at 2, 24, 44 and 64 robots per world, 512 beams and a count that
is not a multiple of 32, on stage 1 (packed inverse lists) and at 0.19 m (plain lists).  And the launch still holds 8
CTAs per SM at the stage-1 and stage-2 shapes."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, make_pair, random_actions
from oracle.oracle import OracleWorld, OrcConfig
from rl_collision_avoidance_b200.scenarios import COMMON, fill_config, make_scenario
from test_env_maps import build_map

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import scatter_work  # noqa: E402

pytestmark = pytest.mark.gpu


def _capacity(name):
    src = open(os.path.join(ROOT, 'rl_collision_avoidance_b200', 'csrc', 'rlca_env.cu')).read()
    return int(re.search(rf'#define {name} (\d+)', src).group(1))


# (map resolution or None = stage 1, robots per world, beams)
CASES = [(None, 2, 512), (None, 24, 512), (None, 44, 500), (None, 64, 512),
         (0.19, 2, 500), (0.19, 24, 500), (0.19, 44, 512), (0.19, 64, 500)]
IDS = [f"{'stage1' if r is None else 'r019'}_R{R}_b{b}" for r, R, b in CASES]


def _pair(res, R, beams, worlds, seed):
    if res is None:
        sc, env, orc = make_pair('stage1', num_worlds=worlds, beams=beams, auto_reset=True, seed=seed,
                                 robots_per_world=R)
        return sc, env, orc
    from rl_collision_avoidance_b200.stage_world import StageWorld
    m = build_map(res, 90, 80, boundary='closed', seed=seed)
    sc = make_scenario('circle', map_=m, robots_per_world=R, radius=6.0)
    ocfg = fill_config(OrcConfig(), sc, num_worlds=worlds, beams=beams, auto_reset=1, seed=seed)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    env = StageWorld(beams, index=0, scenario=sc, num_worlds=worlds, seed=seed, auto_reset=1)
    return sc, env, orc


def _crowded(sc, R, worlds, rng):
    """Per world: the robots on a square grid 0.4 m apart (closer than a footprint: the tick reverts the overlaps),
    round a centre in the map's free space, any heading."""
    m = sc.map
    free_r, free_c = np.nonzero(m.cells == 0)
    ncol = math.ceil(math.sqrt(R))
    pose = np.zeros((worlds * R, 3), np.float32)
    for w in range(worlds):
        k = rng.integers(len(free_r))
        x0 = (free_c[k] - m.origin_cx + 0.5) * m.resolution if w else 0.0
        y0 = (free_r[k] - m.origin_cy + 0.5) * m.resolution if w else 0.0
        for r in range(R):
            pose[w * R + r] = (x0 + 0.4 * (r % ncol - (ncol - 1) / 2), y0 + 0.4 * (r // ncol - (ncol - 1) / 2),
                               rng.uniform(-math.pi, math.pi))
    return pose


def _past_capacity(sc, pose, R, worlds, res):
    """The host model of the CTAs' scatter: the largest queue a CTA asks for, and the fewest long lists (segments) any
    LIDAR_QCAP of its queued cells hold."""
    rc = np.float32(np.float32(1.0 / sc.map.resolution) * np.float32(COMMON['range_max']))
    lens, kr, nslots = scatter_work.list_lengths(rc)
    head = 6 if nslots <= 255 else 4
    assert (res is None) == (nslots <= 255)
    qcap = _capacity('LIDAR_QCAP')
    cells = segs = 0
    for w in range(worlds):
        work = scatter_work.viewer_work(pose[w * R:(w + 1) * R].astype(np.float64), sc.map, lens, kr, head,
                                        COMMON['half_len'], COMMON['half_wid'], COMMON['fov'])
        for rows in scatter_work.cta_rows(work):
            c, s, _ = rows.sum(0)
            cells = max(cells, int(c))
            segs = max(segs, int(s) - max(0, int(c) - qcap))
    return cells, segs


@pytest.mark.parametrize('res,R,beams', CASES, ids=IDS)
def test_pooled_scatter_in_crowded_worlds(built, res, R, beams):
    worlds = 4
    sc, env, orc = _pair(res, R, beams, worlds, seed=11)
    N = orc.N
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(R * 7 + beams)
    pose = _crowded(sc, R, worlds, rng)
    cells, segs = _past_capacity(sc, pose, R, worlds, res)
    print(f'res {res} R={R}: largest queue of a CTA {cells} cells, long lists in any queue-full {segs}')
    if R >= 24:                  # a CTA's four viewers see 23+ robots each: the overflow paths run
        assert cells > _capacity('LIDAR_QCAP') and segs > _capacity('LIDAR_PCAP'), (cells, segs)

    env.control_pose(torch.from_numpy(pose))
    orc.pose[:] = env.state['pose'].cpu().numpy()
    orc.observe()
    assert_outputs_equal(env, orc, f'R={R} crowded: observe')
    p = orc.pose.copy()
    for normalise in (False, True):
        got = env.raycast(torch.from_numpy(p).cuda(), normalise=normalise).cpu().numpy()
        ref = orc.raycast(p, normalise=normalise)
        bad = np.argwhere(got.view(np.uint32) != ref.view(np.uint32))
        assert len(bad) == 0, f'R={R} crowded: raycast (normalise={normalise}) differs for {np.unique(bad[:, 0])[:8]}'
    for t in range(4):
        a = random_actions(rng, N, wide=True)
        env.control_vel(torch.from_numpy(a).cuda())
        orc.step(a)
        assert_state_equal(env, orc, f'R={R} crowded tick {t}')
        assert_outputs_equal(env, orc, f'R={R} crowded tick {t}')
        assert np.array_equal(env.flags.cpu().numpy(), orc.flags), f'R={R} crowded tick {t}: flags differ'
    env.close()


@pytest.mark.parametrize('scenario', ['stage1', 'stage2'])
def test_lidar_launch_holds_8_ctas_per_sm(built, scenario):
    sc, env, _ = make_pair(scenario, num_worlds=2, beams=512, gpu=True)
    n = C.c_int32()
    rc = env.lib.rlca_env_lidar_ctas_per_sm(env._h, C.byref(n))
    assert rc == 0
    print(f'{scenario} (R = {sc.robots_per_world}): {n.value} lidar CTAs per SM')
    assert n.value >= 8
    env.close()
