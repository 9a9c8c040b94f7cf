"""The ORCA-DD controller without a GPU: rlca_orca_action_host (the serial loops over the kernel's per-line code)
against the float64 reference of tests/orca_ref.py on seeded worlds from sparse to packed, and hand cases."""
import numpy as np
import pytest

import orca_ref
from helpers import (ORCA_DT, ORCA_FALLBACK_GAP as FALLBACK_GAP, ORCA_VMAX, ORCA_WMAX, ORCA_WMIN, orca_cfg,
                     orca_sweep_states, orca_world)
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.orca import DEFAULTS, orca_host

DT, VMAX, WMIN, WMAX = ORCA_DT, ORCA_VMAX, ORCA_WMIN, ORCA_WMAX
PARAMS = dict(DEFAULTS)
_cfg = orca_cfg


def _world(rng, R, W, side):
    return orca_world(rng, R, W, side, PARAMS['neighbour_dist'])


CASES = [(1, 4, 8.0), (2, 4, 4.0), (5, 3, 6.0), (24, 3, 12.0), (50, 3, 10.0), (64, 3, 9.0), (64, 2, 5.0)]


def test_orca_host_matches_float64_reference(built):
    rng = np.random.default_rng(20261015)
    p = PARAMS
    seen = {0: 0, 1: 0}
    seen_overlap = seen_ranges = 0
    for R, W, side in CASES:
        pose, goal, meta = _world(rng, R, W, side)
        act, vel, status = orca_host(_cfg(W, R), pose, goal, meta, **p)
        pos, th, _ = orca_ref.agent_state(pose, goal, meta)
        for a in range(R * W):
            P, n = orca_ref.agent_lines(pose, goal, meta, R, a, p['radius'], p['neighbour_dist'], p['time_horizon'], DT)
            if R >= 4 and a % R == 0:
                d = np.hypot(*(pos[a + 2] - pos[a])), np.hypot(*(pos[a + 3] - pos[a]))
                seen_ranges += d[0] < p['neighbour_dist'] < d[1]
            if R >= 2 and a % R == 0:
                seen_overlap += np.hypot(*(pos[a + 1] - pos[a])) < 2 * p['radius']
            vpref = orca_ref.preferred(pos[a], goal[a, 0:2], VMAX, DT)
            v = vel[a].astype(np.float64)
            ref = orca_ref.project(P, n, VMAX, vpref)
            st = int(status[a])
            seen[st] += 1
            if st == 0:
                assert np.hypot(*v) <= VMAX + 1e-5, (R, a)
                assert ref is not None or orca_ref.min_max_penetration(P, n, VMAX)[0] < 1e-4, (R, a)
                if ref is not None:
                    assert np.abs(v - ref).max() <= 1e-4, (R, a, v, ref)
                if len(n):
                    assert orca_ref.penetration(P, n, v).max() <= 1e-5, (R, a)
            else:
                # float32 intersections of nearly parallel projected lines: up to 1.5e-4 outside the speed disk
                assert np.hypot(*v) <= VMAX + 1e-3, (R, a)
                fstar, _ = orca_ref.min_max_penetration(P, n, VMAX)
                assert ref is None or fstar > -1e-4, (R, a, fstar)
                gap = orca_ref.penetration(P, n, v).max() - fstar
                assert -1e-4 <= gap <= FALLBACK_GAP, (R, a, fstar, gap)
            want = orca_ref.track(th[a], v, VMAX, WMIN, WMAX, p['heading_gain'])
            assert np.abs(act[a] - want).max() <= 1e-5, (R, a, act[a], want)
    assert seen[0] > 0 and seen[1] > 0, seen
    assert seen_overlap > 0 and seen_ranges > 0


SWEEP_SEEDS = range(1, 9)


def test_fallback_reaches_least_penetration_on_seeded_sweep(built):
    """Every agent of the packed seeded worlds (helpers.ORCA_SWEEP, seeds 1-8: 4 336 agents, 2 689 of them in the
    least-penetration fallback, up to 63 lines) gets the float64 optimum: status 0 within 1e-4 of the projection,
    status 1 within FALLBACK_GAP of the least max-penetration.  Seed 3 holds the agent whose fallback stopped 0.33 above
    the optimum when the projected lines were anchored at the crossing of the two lines (DESIGN.md §9d).  About 25 s on
    8 CPU cores, mostly in orca_ref.min_max_penetration."""
    p = PARAMS
    fallback = 0
    for (seed, R, W, side), (pose, goal, meta) in orca_sweep_states(SWEEP_SEEDS, p['neighbour_dist']):
        _, vel, status = orca_host(_cfg(W, R), pose, goal, meta, **p)
        pos, _, _ = orca_ref.agent_state(pose, goal, meta)
        for a in range(R * W):
            P, n = orca_ref.agent_lines(pose, goal, meta, R, a, p['radius'], p['neighbour_dist'], p['time_horizon'], DT)
            v = vel[a].astype(np.float64)
            if status[a] == 0:
                ref = orca_ref.project(P, n, VMAX, orca_ref.preferred(pos[a], goal[a, 0:2], VMAX, DT))
                assert ref is not None and np.abs(v - ref).max() <= 1e-4, (seed, R, side, a, v, ref)
                continue
            gap = orca_ref.penetration(P, n, v).max() - orca_ref.min_max_penetration(P, n, VMAX)[0]
            assert -1e-4 <= gap <= FALLBACK_GAP, (seed, R, side, a, len(n), gap)
            fallback += 1
    assert fallback >= 2500, fallback


def _state(xy, th, v, goal_xy, stalled=None):
    n = len(xy)
    pose = np.zeros((n, 4), np.float32)
    goal = np.zeros((n, 4), np.float32)
    meta = np.zeros((n, 4), np.int32)
    pose[:, 0:2], pose[:, 2] = xy, th
    goal[:, 0:2], goal[:, 2] = goal_xy, v
    if stalled is not None:
        meta[:, 2] = stalled
    return pose, goal, meta


def test_lone_robot_gets_preferred_velocity(built):
    pose, goal, meta = _state([[0.0, 0.0]], [0.0], [0.5], [[3.0, 4.0]])
    act, vel, st = orca_host(_cfg(1, 1), pose, goal, meta, **PARAMS)
    assert st[0] == 0 and np.allclose(vel[0], [0.6, 0.8], atol=1e-6)
    # 0.05 m from the goal: v_pref = d / dt, below v_max
    pose, goal, meta = _state([[1.0, 1.0]], [0.0], [0.0], [[1.03, 1.04]])
    act, vel, st = orca_host(_cfg(1, 1), pose, goal, meta, **PARAMS)
    assert np.allclose(vel[0], [0.3, 0.4], atol=1e-5)
    assert np.isclose(act[0, 0], 0.3, atol=1e-5)
    assert np.isclose(act[0, 1], min(PARAMS['heading_gain'] * 0.8, WMAX), atol=1e-5)
    # on the goal: no motion
    pose, goal, meta = _state([[1.0, 1.0]], [0.0], [0.7], [[1.0, 1.0]])
    act, vel, st = orca_host(_cfg(1, 1), pose, goal, meta, **PARAMS)
    assert np.all(vel[0] == 0) and np.all(act[0] == 0)


def test_head_on_pair_is_point_symmetric(built):
    pose, goal, meta = _state([[-2.0, 0.0], [2.0, 0.0]], [0.0, np.pi], [1.0, 1.0], [[4.0, 0.0], [-4.0, 0.0]])
    act, vel, st = orca_host(_cfg(1, 2), pose, goal, meta, **PARAMS)
    assert np.all(st == 0)
    assert np.abs(vel[0] + vel[1]).max() <= 1e-6, vel
    assert abs(vel[0, 1]) > 0.05                                    # they do swerve
    assert np.abs(act[0] - act[1]).max() <= 1e-5, act               # same (v, w) in each robot's own frame


def test_robot_facing_away_turns_in_place(built):
    for gy, w in ((0.5, WMAX), (-0.5, WMIN)):
        pose, goal, meta = _state([[0.0, 0.0]], [0.0], [0.0], [[-5.0, gy]])
        act, _, _ = orca_host(_cfg(1, 1), pose, goal, meta, **PARAMS)
        assert act[0, 0] == 0.0 and act[0, 1] == np.float32(w)


def test_stalled_neighbour_has_no_velocity(built):
    """A stalled neighbour's last command does not count: same answer as a neighbour commanded v = 0."""
    xy, th, g = [[0.0, 0.0], [1.5, 0.2]], [0.0, np.pi], [[5.0, 0.0], [-5.0, 0.0]]
    a = orca_host(_cfg(1, 2), *_state(xy, th, [0.8, 0.9], g, stalled=[0, 1]), **PARAMS)
    b = orca_host(_cfg(1, 2), *_state(xy, th, [0.8, 0.0], g), **PARAMS)
    assert np.array_equal(a[0][0], b[0][0]) and np.array_equal(a[1][0], b[1][0])


@pytest.mark.parametrize('bad', [dict(radius=0.0), dict(neighbour_dist=-1.0), dict(time_horizon=float('inf')),
                                 dict(heading_gain=float('nan'))])
def test_bad_parameters_raise(built, bad):
    pose, goal, meta = _state([[0.0, 0.0]], [0.0], [0.0], [[1.0, 0.0]])
    with pytest.raises(_lib.RlcaError):
        orca_host(_cfg(1, 1), pose, goal, meta, **{**PARAMS, **bad})
    cfg = _cfg(1, 1)
    cfg.v_max = 0.0
    with pytest.raises(_lib.RlcaError):
        orca_host(cfg, pose, goal, meta, **PARAMS)
