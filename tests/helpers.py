"""Shared helpers for the parity tests: build a GPU StageWorld and its oracle twin; the ORCA-DD tests' states and
configs, and a replica of the ORCA kernel's incremental LPs."""
import numpy as np

from oracle.oracle import OracleWorld, OrcConfig
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario


def make_pair(scenario='stage1', num_worlds=3, beams=512, auto_reset=True, seed=0, ctas_per_world=0,
              world_offset=0, raw_beams=None, gpu=True, robots_per_world=None, radius=None, max_reject=4096):
    """`robots_per_world` and `radius` reshape stage 1 / circle (make_scenario); `max_reject` is the spawn sampler's
    try budget."""
    sc = make_scenario(scenario, robots_per_world=robots_per_world, radius=radius)
    ocfg = fill_config(OrcConfig(), sc, num_worlds=num_worlds, beams=beams, raw_beams=raw_beams,
                       auto_reset=auto_reset, seed=seed, world_offset=world_offset, max_reject=max_reject)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    env = None
    if gpu:
        from rl_collision_avoidance_b200.stage_world import StageWorld
        env = StageWorld(beams, index=0, scenario=sc, num_worlds=num_worlds, seed=seed, auto_reset=auto_reset,
                         ctas_per_world=ctas_per_world, world_offset=world_offset, raw_beams=raw_beams,
                         max_reject=max_reject)
    return sc, env, orc


def random_actions(rng, n, wide=False):
    lo, hi = (-0.3, 1.3) if wide else (0.0, 1.0)
    a = np.stack([rng.uniform(lo, hi, n), rng.uniform(-1.3 if wide else -1.0, 1.3 if wide else 1.0, n)], 1)
    return a.astype(np.float32)


# ---------------------------------------------------------------------------------------------- ORCA-DD (DESIGN.md §9d)
ORCA_DT, ORCA_VMAX, ORCA_WMIN, ORCA_WMAX = 0.1, 1.0, -1.0, 1.0
# largest max-penetration a least-penetration (status 1) velocity may have above the float64 optimum, for every agent;
# the worst measured on the seeded sweep is 6.1e-7, from the float32 half-planes alone
ORCA_FALLBACK_GAP = 1e-4


def orca_cfg(worlds, robots, dt=ORCA_DT):
    """The EnvConfig fields rlca_orca_action reads."""
    from rl_collision_avoidance_b200 import _lib
    c = _lib.EnvConfig()
    c.robots_per_world, c.num_worlds = robots, worlds
    c.dt, c.inv_dt = dt, np.float32(1.0) / np.float32(dt)
    c.v_min, c.v_max, c.w_min, c.w_max = 0.0, ORCA_VMAX, ORCA_WMIN, ORCA_WMAX
    return c


def orca_world(rng, R, W, side, neighbour_dist):
    """W worlds of R robots in a side x side box: random headings and last commands, some stalled robots and some on
    their goals; world 0 also gets an overlapping pair and neighbours just inside / outside neighbour_dist."""
    n = R * W
    pose = np.zeros((n, 4), np.float32)
    goal = np.zeros((n, 4), np.float32)
    meta = np.zeros((n, 4), np.int32)
    pose[:, 0:2] = rng.uniform(-side / 2, side / 2, (n, 2))
    pose[:, 2] = rng.uniform(-np.pi, np.pi, n)
    goal[:, 0:2] = rng.uniform(-10, 10, (n, 2))
    goal[:, 2] = rng.uniform(0, ORCA_VMAX, n)
    goal[:, 3] = rng.uniform(ORCA_WMIN, ORCA_WMAX, n)
    meta[:, 2] = rng.random(n) < 0.15
    on_goal = rng.random(n) < 0.1
    goal[on_goal, 0:2] = pose[on_goal, 0:2]
    nd = neighbour_dist
    if R >= 2:
        pose[1, 0:2] = pose[0, 0:2] + np.float32([0.3, 0.2])                       # overlap: the one-step branch
    if R >= 4:
        far = np.float32([np.cos(0.7), np.sin(0.7)])
        pose[2, 0:2] = pose[0, 0:2] + (nd - 1e-3) * far                             # just inside
        pose[3, 0:2] = pose[0, 0:2] - (nd + 1e-3) * far                             # just outside
    return pose, goal, meta


# The packed worlds of the fallback sweep (R, W, side): orca_world(np.random.default_rng(seed), *case) in this order
ORCA_SWEEP = [(24, 3, 12.0), (50, 3, 10.0), (64, 3, 9.0), (64, 2, 5.0)]


def orca_sweep_states(seeds, neighbour_dist):
    for seed in seeds:
        rng = np.random.default_rng(seed)
        for R, W, side in ORCA_SWEEP:
            yield (seed, R, W, side), orca_world(rng, R, W, side, neighbour_dist)


def orca_lp_trace(P, n, vmax, vpref, eps=1e-5):
    """Float64 replica of the structure of the ORCA kernel's incremental LPs (csrc/rlca_orca.cu: lp2 / lp3, same line
    order, branches and parallel threshold) on the half-planes (P, n) of orca_ref.agent_lines.  Returns the velocity,
    the first line the 2-D LP fails on (len(n) when feasible), the violated lines the 2-D LP solved, and per line the
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
        proj = []
        for qx, qy, ex, ey in L[:i]:
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
    return dict(v=np.array([rx, ry]), fail=fail, solved=solved, lp3=passes)


def assert_state_equal(env, orc, tag=''):
    import torch
    torch.cuda.synchronize()
    st = env.state
    for k, ref in (('pose', orc.pose), ('goal', orc.goal), ('acc', orc.acc), ('meta', orc.meta)):
        got = st[k].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), f'{tag}: state {k} differs at rows ' \
            f'{np.unique(np.nonzero(got.view(np.uint32) != ref.view(np.uint32))[0])[:8]}'


def assert_outputs_equal(env, orc, tag='', obs=None):
    import torch
    torch.cuda.synchronize()
    o = (env.obs if obs is None else obs).cpu().numpy()
    assert np.array_equal(o.view(np.uint32), orc.obs.view(np.uint32)), \
        f'{tag}: obs differ, max abs {np.abs(o - orc.obs).max()} at {np.argwhere(o != orc.obs)[:4]}'
    assert np.array_equal(env.gs.cpu().numpy().view(np.uint32), orc.gs.view(np.uint32)), f'{tag}: gs differ'
