"""The NH-ORCA controller without a GPU (DESIGN.md §9e): the velocity polygon P, rlca_nh_orca_action_host against the
float64 reference of tests/nh_orca_ref.py on seeded worlds from sparse to packed, the arc tracker, and hand cases."""
import numpy as np
import pytest

import nh_orca_ref as ref
import orca_ref
from helpers import ORCA_DT, ORCA_VMAX, ORCA_WMAX, ORCA_WMIN, orca_cfg, orca_sweep_states, orca_world
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.orca import NH_DEFAULTS, NH_ORCA_VERTS, nh_orca_host, nh_orca_polygon

DT, VMIN, VMAX, WMIN, WMAX = ORCA_DT, 0.0, ORCA_VMAX, ORCA_WMIN, ORCA_WMAX
PARAMS = dict(NH_DEFAULTS)
E, T = PARAMS['tracking_error'], PARAMS['heading_time']


def _polygon_area(v):
    return 0.5 * float(np.sum(v[:, 0] * np.roll(v[:, 1], -1) - v[:, 1] * np.roll(v[:, 0], -1)))


def test_tracking_error_closed_form():
    """The measured largest distance of the arc tracker from the holonomic trajectory is V T_th |sin(th/2)|."""
    rng = np.random.default_rng(3)
    for V, th, T_ in zip(rng.uniform(0, 1, 40), rng.uniform(-np.pi, np.pi, 40), rng.choice([0.1, 0.4, 1.5], 40)):
        want = V * float(ref.turn_time(th, T_, WMIN, WMAX)) * abs(np.sin(th / 2))
        assert abs(ref.tracking_error(V, th, T_, WMIN, WMAX) - want) <= 1e-12, (V, th, T_)


@pytest.mark.parametrize('E_', [0.01, 0.05, 0.2])
@pytest.mark.parametrize('T_', [0.1, 0.4, 1.5])
def test_polygon_inside_trackable_set(built, E_, T_):
    v = nh_orca_polygon(orca_cfg(1, 1), E_, T_).astype(np.float64)
    k = len(v)
    assert 3 <= k <= NH_ORCA_VERTS
    d = np.roll(v, -1, 0) - v
    turn = d[:, 0] * np.roll(d, -1, 0)[:, 1] - d[:, 1] * np.roll(d, -1, 0)[:, 0]
    assert turn.min() > 0                                                       # convex, counter-clockwise
    inradius = ((v[:, 0] * d[:, 1] - v[:, 1] * d[:, 0]) / np.hypot(d[:, 0], d[:, 1])).min()
    assert inradius > 0.1 * E_, inradius                                        # origin strictly inside
    # every point of every edge: tracking error <= E, v* <= v_max, |w| within bounds
    q = (v[:, None, :] + np.linspace(0, 1, 1000)[None, :, None] * d[:, None, :]).reshape(-1, 2)
    V, th = np.hypot(q[:, 0], q[:, 1]), np.arctan2(q[:, 1], q[:, 0])
    turn_t = ref.turn_time(th, T_, WMIN, WMAX)
    assert np.all(V * turn_t * np.abs(np.sin(th / 2)) <= E_ * (1 + 1e-6))
    assert np.all(ref.arc_speed(V, th) <= VMAX)
    w = th / turn_t
    assert np.all((w >= WMIN) & (w <= WMAX))
    # the measured error, at the points of largest closed-form error of each edge
    eps = (V * turn_t * np.abs(np.sin(th / 2))).reshape(k, 1000)
    for e in range(k):
        j = e * 1000 + int(np.argmax(eps[e]))
        assert ref.tracking_error(V[j], th[j], T_, WMIN, WMAX) <= E_ * (1 + 1e-6)
    # area against S_E's
    a = np.linspace(-np.pi, np.pi, 200001)
    s_area = 0.5 * np.trapezoid(ref.speed_bound(a, E_, T_, VMAX, WMIN, WMAX) ** 2, a)
    assert _polygon_area(v) >= 0.85 * s_area, _polygon_area(v) / s_area


# status-0 velocities: within 1e-6 m/s of the float64 optimum for at least 99 % of the agents, and STATUS0_TOL for all.
# The worst measured, 2.6e-6 for one of 573, sits where an ORCA line crosses an edge of P at a small angle, which
# magnifies the float32 rounding of both lines.
STATUS0_TOL = 5e-6


def _assert_status0_close(outs):
    errs = np.array([o['err'] for o in outs if o['status'] == 0])
    assert np.mean(errs <= 1e-6) >= 0.99, np.sort(errs)[-5:]


def nh_lp_trace(P, n, hard, vmax, vpref, eps=1e-5):
    """Float64 replica of the structure of the NH-ORCA kernel's incremental LPs (csrc/rlca_orca.cu: lp2 / lp3 with
    the first `hard` lines hard, same line order, branches and parallel threshold) on half-planes (P, n), P's first.
    Returns the first line the 2-D LP fails on (len(n) when feasible), the violated lines it solved, and per line the
    least-penetration program passes over: (line, projected lines, projected line the inner LP failed on, violated
    projected lines)."""
    L = [(float(p[0]), float(p[1]), float(m[1]), -float(m[0])) for p, m in zip(P, n)]   # point, unit direction

    def det(ax, ay, bx, by):
        return ax * by - ay * bx

    def lp2(lines, ox, oy, dir_opt):
        if dir_opt:
            rx, ry = ox * vmax, oy * vmax
        else:
            s = min(1.0, vmax / max(np.hypot(ox, oy), 1e-300))
            rx, ry = ox * s, oy * s
        solved = []
        for i, (px, py, dx, dy) in enumerate(lines):
            if not det(dx, dy, px - rx, py - ry) > 0:
                continue
            solved.append(i)
            dot = px * dx + py * dy
            disc = dot * dot + vmax * vmax - (px * px + py * py)
            if disc < 0:
                return i, rx, ry, solved
            tl, tr = -dot - np.sqrt(disc), -dot + np.sqrt(disc)
            for qx, qy, ex, ey in lines[:i]:
                den, num = det(dx, dy, ex, ey), det(ex, ey, px - qx, py - qy)
                if abs(den) <= eps:
                    if num < 0:
                        return i, rx, ry, solved
                elif den >= 0:
                    tr = min(tr, num / den)
                else:
                    tl = max(tl, num / den)
            if tl > tr:
                return i, rx, ry, solved
            if dir_opt:
                t = tr if ox * dx + oy * dy > 0 else tl
            else:
                t = min(max(dx * (ox - px) + dy * (oy - py), tl), tr)
            rx, ry = px + t * dx, py + t * dy
        return len(lines), rx, ry, solved

    fail, rx, ry, solved = lp2(L, float(vpref[0]), float(vpref[1]), False)
    passes, dist = [], 0.0
    for i in range(fail, len(L)):
        px, py, dx, dy = L[i]
        if not det(dx, dy, px - rx, py - ry) > dist:
            continue
        proj = list(L[:hard])
        for qx, qy, ex, ey in L[hard:i]:
            if abs(det(dx, dy, ex, ey)) <= eps and dx * ex + dy * ey > 0:
                continue
            gx, gy = ex - dx, ey - dy
            k = det(ex, ey, qx - px, qy - py) / (gx * gx + gy * gy)
            gl = np.hypot(gx, gy)
            proj.append((px - k * gy, py + k * gx, gx / gl, gy / gl))
        f, qx, qy, psolved = lp2(proj, -dy, dx, True)
        passes.append((i, len(proj), f, psolved))
        if f == len(proj):
            rx, ry = qx, qy
        dist = det(dx, dy, px - rx, py - ry)
    return dict(fail=fail, solved=solved, lp3=passes)


def check_agents(R, W, pose, goal, meta, vel, status, act, p=PARAMS, trace=False):
    """Every agent against the float64 reference: status 0 within STATUS0_TOL m/s of the projection onto the ORCA
    lines and P, status 1 inside P and within 1e-4 of the least largest ORCA penetration over P; the action is the
    tracker's for the returned velocity, and that arc stays within E of the holonomic trajectory.  Returns per agent
    the line count, status, status-0 distance 'err' and (with `trace`) the replica's trace."""
    verts = nh_orca_polygon(orca_cfg(W, R), p['tracking_error'], p['heading_time'])
    pos, th, _ = orca_ref.agent_state(pose, goal, meta)
    out = []
    for a in range(R * W):
        P, n = orca_ref.agent_lines(pose, goal, meta, R, a, p['radius'] + p['tracking_error'], p['neighbour_dist'],
                                    p['time_horizon'], DT)
        Ph, nh = ref.polygon_half_planes(verts, th[a])
        vpref = orca_ref.preferred(pos[a], goal[a, 0:2], VMAX, DT)
        v = vel[a].astype(np.float64)
        if status[a] == 0:
            want = ref.project(P, n, Ph, nh, VMAX, vpref)
            err = np.abs(v - want).max() if want is not None else np.inf
            assert err <= STATUS0_TOL, (R, a, v, want)
        else:
            assert len(n) and orca_ref.penetration(Ph, nh, v).max() <= 1e-6, (R, a)
            fstar, _ = ref.least_penetration(P, n, Ph, nh)
            gap = orca_ref.penetration(P, n, v).max() - fstar
            assert abs(gap) <= 1e-4, (R, a, len(n), gap)
        want, (V, ang, turn) = ref.track(th[a], v, VMIN, VMAX, WMIN, WMAX, p['heading_time'])
        assert np.abs(act[a] - want).max() <= 1e-5, (R, a, act[a], want)
        if V > 1e-6:
            dev = ref.deviation(float(act[a, 0]), float(act[a, 1]), turn, V, ang, steps=201)
            assert dev <= p['tracking_error'] + 1e-5, (R, a, dev)
        o = dict(lines=len(n), status=int(status[a]), err=err if status[a] == 0 else 0.0)
        if trace:
            o['trace'] = nh_lp_trace(np.concatenate((Ph, P)), np.concatenate((nh, n)), len(Ph), VMAX, vpref)
        out.append(o)
    return out


CASES = [(1, 4, 8.0), (2, 4, 4.0), (5, 3, 6.0), (24, 3, 12.0), (50, 3, 10.0), (64, 3, 9.0), (64, 2, 5.0)]


def test_nh_orca_host_matches_float64_reference(built):
    rng = np.random.default_rng(20261015)
    outs = []
    for R, W, side in CASES:
        pose, goal, meta = orca_world(rng, R, W, side, PARAMS['neighbour_dist'])
        act, vel, status = nh_orca_host(orca_cfg(W, R), pose, goal, meta, **PARAMS)
        outs += check_agents(R, W, pose, goal, meta, vel, status, act)
    _assert_status0_close(outs)
    assert {o['status'] for o in outs} == {0, 1}


def test_seeded_sweep_reaches_third_lane_stride(built):
    """The packed seeded worlds (helpers.ORCA_SWEEP, seeds 1-4) against the reference, agent by agent.  With P's 32
    lines first the lists hold up to 95 lines, so the sweep must reach the lanes' third stride: a first failing line
    >= 64, violated lines >= 64 (the bound scan) and fallback passes over lines >= 64 (the third ballot-compaction
    pass), counted with the float64 replica of the incremental LPs."""
    outs = []
    for (seed, R, W, side), (pose, goal, meta) in orca_sweep_states(range(1, 5), PARAMS['neighbour_dist']):
        act, vel, status = nh_orca_host(orca_cfg(W, R), pose, goal, meta, **PARAMS)
        outs += check_agents(R, W, pose, goal, meta, vel, status, act, trace=True)
    _assert_status0_close(outs)
    fallback = [o for o in outs if o['status']]
    assert all((o['trace']['fail'] < o['lines'] + NH_ORCA_VERTS) == o['status'] for o in outs)
    assert all(o['trace']['fail'] >= NH_ORCA_VERTS for o in fallback)          # P alone is always feasible
    assert fallback and len(fallback) < len(outs)
    assert sum(o['trace']['fail'] >= 64 for o in fallback) >= 5
    assert sum(max(o['trace']['solved'], default=0) >= 64 for o in outs) >= 5
    assert sum(any(i >= 64 for i, *_ in o['trace']['lp3']) for o in fallback) >= 5


def _state(xy, th, v, goal_xy):
    n = len(xy)
    pose = np.zeros((n, 4), np.float32)
    goal = np.zeros((n, 4), np.float32)
    meta = np.zeros((n, 4), np.int32)
    pose[:, 0:2], pose[:, 2] = xy, th
    goal[:, 0:2], goal[:, 2] = goal_xy, v
    return pose, goal, meta


def test_lone_robot_gets_preferred_velocity_clipped_to_polygon(built):
    for heading, g in ((0.0, [3.0, 4.0]), (0.3, [3.0, 0.0]), (2.0, [-1.0, 2.0]), (0.0, [0.03, 0.04]), (0.0, [5.0, 0.0])):
        pose, goal, meta = _state([[0.0, 0.0]], [heading], [0.5], [g])
        act, vel, st = nh_orca_host(orca_cfg(1, 1), pose, goal, meta, **PARAMS)
        Ph, nh = ref.polygon_half_planes(nh_orca_polygon(orca_cfg(1, 1), E, T), heading)
        want = ref.project(np.zeros((0, 2)), np.zeros((0, 2)), Ph, nh, VMAX,
                           orca_ref.preferred(np.zeros(2), np.array(g), VMAX, DT))
        assert st[0] == 0 and np.abs(vel[0] - want).max() <= 1e-6, (heading, vel[0], want)
    # on the goal: no motion
    pose, goal, meta = _state([[1.0, 1.0]], [0.0], [0.7], [[1.0, 1.0]])
    act, vel, st = nh_orca_host(orca_cfg(1, 1), pose, goal, meta, **PARAMS)
    assert np.all(vel[0] == 0) and np.all(act[0] == 0)


def test_head_on_pair_is_point_symmetric(built):
    pose, goal, meta = _state([[-2.0, 0.0], [2.0, 0.0]], [0.0, np.pi], [1.0, 1.0], [[4.0, 0.0], [-4.0, 0.0]])
    act, vel, st = nh_orca_host(orca_cfg(1, 2), pose, goal, meta, **PARAMS)
    assert np.abs(vel[0] + vel[1]).max() <= 1e-6, vel
    assert abs(vel[0, 1]) > 0.01                                    # they do swerve
    assert np.abs(act[0] - act[1]).max() <= 1e-5, act               # same (v, w) in each robot's own frame


def test_goal_behind_turns_at_full_rate(built):
    """A goal straight behind: the velocity chosen is near the back of P, |th| >= T w_max, so th / T_th = +-w_max, and
    the speed of the arc is almost 0."""
    for gy in (0.0, 0.02, -0.02):
        pose, goal, meta = _state([[0.0, 0.0]], [0.0], [0.0], [[-5.0, gy]])
        act, _, _ = nh_orca_host(orca_cfg(1, 1), pose, goal, meta, **PARAMS)
        assert abs(abs(act[0, 1]) - WMAX) <= 1e-6 and 0.0 <= act[0, 0] <= 0.01, act[0]


@pytest.mark.parametrize('bad', [dict(radius=0.0), dict(neighbour_dist=-1.0), dict(time_horizon=float('inf')),
                                 dict(tracking_error=float('nan')), dict(tracking_error=0.0),
                                 dict(heading_time=-0.4), dict(heading_time=float('inf'))])
def test_bad_parameters_raise(built, bad):
    pose, goal, meta = _state([[0.0, 0.0]], [0.0], [0.0], [[1.0, 0.0]])
    with pytest.raises(_lib.RlcaError):
        nh_orca_host(orca_cfg(1, 1), pose, goal, meta, **{**PARAMS, **bad})


@pytest.mark.parametrize('field, value', [('v_max', 0.0), ('v_min', 0.1), ('w_min', 0.0), ('w_max', 0.0),
                                          ('w_max', float('nan'))])
def test_bad_config_raises(built, field, value):
    pose, goal, meta = _state([[0.0, 0.0]], [0.0], [0.0], [[1.0, 0.0]])
    cfg = orca_cfg(1, 1)
    setattr(cfg, field, value)
    with pytest.raises(_lib.RlcaError):
        nh_orca_host(cfg, pose, goal, meta, **PARAMS)
    with pytest.raises(_lib.RlcaError):
        nh_orca_polygon(cfg, E, T)


def test_evaluate_py_rejects_orca_gain_with_nh_orca(built):
    import evaluate as drv
    with pytest.raises(SystemExit):
        drv.main(['--scenario', 'stage1', '--baseline', 'nh-orca', '--orca-gain', '2'])
