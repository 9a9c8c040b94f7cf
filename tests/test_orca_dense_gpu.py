"""The ORCA-DD kernel on the H100 against the float64 reference (tests/orca_ref.py) on constructed states: every robot
count from 1 to 64 in packed worlds where an agent sees all R - 1 others, agent counts that leave the last CTA partly
empty, degenerate geometry and parameter edges, and the seeded fallback sweep of tests/test_orca.py.  Every case
requires action, velocity and status equal to rlca_orca_action_host bit for bit, every status-0 velocity within 1e-4 of
the projection and every status-1 velocity within ORCA_FALLBACK_GAP of the least max-penetration, and asserts that it
reached what it targets, counted with the replica of the incremental LPs in helpers.orca_lp_trace."""
import ctypes as C

import numpy as np
import pytest
import torch

import orca_ref
from helpers import (ORCA_DT, ORCA_FALLBACK_GAP, ORCA_VMAX, ORCA_WMAX, ORCA_WMIN, orca_cfg, orca_lp_trace,
                     orca_sweep_states)
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.orca import DEFAULTS, orca_host

pytestmark = pytest.mark.gpu


def _device(cfg, pose, goal, meta, p):
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in (('pose', pose), ('goal', goal),
                                                                             ('meta', meta))}
    acc = torch.zeros_like(dev['pose'])
    st = _lib.EnvState(dev['pose'].data_ptr(), dev['goal'].data_ptr(), acc.data_ptr(), dev['meta'].data_ptr())
    n = len(pose)
    act = torch.full((n, 2), float('nan'), device='cuda')
    vel = torch.full((n, 2), float('nan'), device='cuda')
    status = torch.full((n,), -1, dtype=torch.int32, device='cuda')
    ptr = lambda t: C.c_void_p(t.data_ptr())
    _lib.check(_lib.load().rlca_orca_action(C.byref(cfg), C.byref(st), p['radius'], p['neighbour_dist'],
                                            p['time_horizon'], p['heading_gain'], ptr(act), ptr(vel), ptr(status),
                                            None))
    torch.cuda.synchronize()
    return act.cpu().numpy(), vel.cpu().numpy(), status.cpu().numpy()


def _check(R, W, pose, goal, meta, p=None, dt=ORCA_DT, reference=True):
    """Device against host bit for bit and, with `reference`, every agent against the float64 optimum.  Returns per
    agent the line count, status and replica trace."""
    p = dict(DEFAULTS, **(p or {}))
    cfg = orca_cfg(W, R, dt)
    d_act, d_vel, d_st = _device(cfg, pose, goal, meta, p)
    h_act, h_vel, h_st = orca_host(cfg, pose, goal, meta, **p)
    assert np.array_equal(d_act.view(np.uint32), h_act.view(np.uint32))
    assert np.array_equal(d_vel.view(np.uint32), h_vel.view(np.uint32))
    assert np.array_equal(d_st, h_st)
    if not reference:
        return None
    pos, th, _ = orca_ref.agent_state(pose, goal, meta)
    out = []
    for a in range(R * W):
        P, n = orca_ref.agent_lines(pose, goal, meta, R, a, p['radius'], p['neighbour_dist'], p['time_horizon'], dt)
        vpref = orca_ref.preferred(pos[a], goal[a, 0:2], ORCA_VMAX, dt)
        v = h_vel[a].astype(np.float64)
        # float32 half-planes round in proportion to their size: 40 m/s when a 8 m wide pair overlaps at dt = 0.1 s
        scale = max(1.0, np.abs(P).max(initial=0.0))
        if h_st[a] == 0:
            ref = orca_ref.project(P, n, ORCA_VMAX, vpref)
            assert ref is not None and np.abs(v - ref).max() <= 1e-4 * scale, (R, a, v, ref)
        else:
            gap = orca_ref.penetration(P, n, v).max() - orca_ref.min_max_penetration(P, n, ORCA_VMAX)[0]
            assert abs(gap) <= ORCA_FALLBACK_GAP * scale, (R, a, len(n), gap)
        want = orca_ref.track(th[a], v, ORCA_VMAX, ORCA_WMIN, ORCA_WMAX, p['heading_gain'])
        assert np.abs(h_act[a] - want).max() <= 1e-5, (R, a, h_act[a], want)
        out.append(dict(lines=len(n), status=int(h_st[a]), trace=orca_lp_trace(P, n, ORCA_VMAX, vpref)))
    return out


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


def _packed(rng, R, W, side, inner):
    """W worlds of R robots: robots 0-31 of each world in a side x side box, robots 32 on in an inner x inner box at
    its centre, so that an agent of the inner box meets its closest neighbours from line 32 on."""
    n = R * W
    r = np.arange(n) % R
    half = np.where(r < 32, side, inner)[:, None] / 2
    xy = rng.uniform(-1, 1, (n, 2)) * half                  # worlds overlap: a wrong world base adds lines
    pose, goal, meta = _state(xy, rng.uniform(-np.pi, np.pi, n), rng.uniform(0, ORCA_VMAX, n),
                              xy + rng.uniform(-10, 10, (n, 2)))
    return pose, goal, meta


# (R, W, side, inner): R * W is not a multiple of the 8 agents of a CTA except at R = 32 and 64
ROBOT_COUNTS = [(1, 5, 1.0, 1.0), (2, 3, 1.0, 1.0), (3, 5, 1.5, 1.5), (31, 3, 4.0, 4.0), (32, 1, 4.0, 4.0),
                (33, 3, 4.0, 4.0), (34, 3, 6.0, 2.0), (63, 2, 6.0, 3.0), (64, 2, 6.0, 3.0)]


@pytest.mark.parametrize('R, W, side, inner', ROBOT_COUNTS)
def test_packed_worlds_every_agent_sees_every_robot(built, R, W, side, inner):
    pose, goal, meta = _packed(np.random.default_rng(R), R, W, side, inner)
    out = _check(R, W, pose, goal, meta, dict(neighbour_dist=2 * side))
    assert all(o['lines'] == R - 1 for o in out)
    fallback = [o for o in out if o['status']]
    assert all((o['trace']['fail'] < o['lines']) == o['status'] for o in out)     # the replica takes the same branch
    if R >= 3:
        assert fallback and len(fallback) < R * W, len(fallback)
    if R >= 63:
        # the lanes' second stride of the bound scan (a violated line >= 33, in the 2-D LP and in a projected one),
        # the second ballot-compaction pass of the projected lines (a fallback pass over a line >= 33)
        assert sum(o['trace']['fail'] >= 33 for o in fallback) >= 5
        assert sum(max(o['trace']['solved'], default=0) >= 33 for o in out) >= 5
        assert sum(any(i >= 33 for i, *_ in o['trace']['lp3']) for o in fallback) >= 20
        assert sum(any(k >= 33 for *_, solved in o['trace']['lp3'] for k in solved) for o in fallback) >= 20


def test_degenerate_geometry(built):
    # 0: two neighbours with identical pose and velocity (identical lines), then a mirrored head-on pair of each side
    # of it (antiparallel one-tick-disk lines: the fallback), a stalled neighbour and an agent on its goal
    xy = [[0.0, 0.0], [1.0, 0.25], [1.0, 0.25], [-0.5, 0.0], [0.5, 0.0], [0.0, -1.0], [2.0, 2.0]]
    th = [0.0, np.pi, np.pi, 0.0, np.pi, np.pi / 2, 0.0]
    v = [0.8, 0.6, 0.6, 0.9, 0.9, 0.7, 0.5]
    goals = [[5.0, 0.0], [-5.0, 0.0], [-5.0, 0.0], [5.0, 0.0], [-5.0, 0.0], [0.0, 5.0], [2.0, 2.0]]
    pose, goal, meta = _state(xy, th, v, goals, stalled=[0, 0, 0, 0, 0, 1, 0])
    out = _check(1, 7, pose, goal, meta) + _check(7, 1, pose, goal, meta)
    assert out[-7]['status'] == 1 and out[-7]['lines'] == 6                    # agent 0 of the 7-robot world
    assert np.all(goal[6, 0:2] == pose[6, 0:2])
    # 1: relative velocity exactly at the centre of the one-tick disk (dt = 1/8): neither robot gets a line
    pose, goal, meta = _state([[0.0, 0.0], [0.125, 0.0]], [0.0, 0.0], [1.0, 0.0], [[3.0, 0.0], [-3.0, 0.0]])
    out = _check(2, 1, pose, goal, meta, dt=0.125)
    assert [o['lines'] for o in out] == [0, 0]
    # 2: neighbours at exactly neighbour_dist (not neighbours), and just inside
    xy = [[0.0, 0.0], [3.0, 4.0], [0.0, -5.0], [-4.0, -3.0], [-2.0, 4.5]]
    pose, goal, meta = _state(xy, [0.0, 1.0, 2.0, 3.0, -1.0], [0.5] * 5, [[-1.0, 1.0]] * 5)
    out = _check(5, 1, pose, goal, meta, dict(neighbour_dist=5.0))
    assert out[0]['lines'] == 1


def test_parameter_edges(built):
    rng = np.random.default_rng(7)
    pose, goal, meta = _packed(rng, 24, 3, 4.0, 4.0)
    # time_horizon = dt: the cut-off arc is the one-tick disk
    out = _check(24, 3, pose, goal, meta, dict(neighbour_dist=8.0, time_horizon=ORCA_DT))
    assert all(o['lines'] == 23 for o in out)
    # a radius so large that every pair overlaps: only the one-tick-disk branch
    _check(24, 3, pose, goal, meta, dict(neighbour_dist=8.0, radius=4.0))
    # neighbour_dist below the closest pair: no lines, every agent gets its preferred velocity
    gaps = [np.hypot(*(pose[a, 0:2] - pose[b, 0:2])) for w in range(3) for a in range(24 * w, 24 * w + 24)
            for b in range(a + 1, 24 * w + 24)]
    out = _check(24, 3, pose, goal, meta, dict(neighbour_dist=0.5 * min(gaps)))
    assert all(o['lines'] == 0 and o['status'] == 0 for o in out)


def test_seeded_fallback_sweep_on_device(built):
    """The states of tests/test_orca.py's seeded sweep (which checks the host against the float64 reference): the
    device equals the host bit for bit on all of them."""
    for (seed, R, W, side), (pose, goal, meta) in orca_sweep_states(range(1, 9), DEFAULTS['neighbour_dist']):
        _check(R, W, pose, goal, meta, reference=False)
