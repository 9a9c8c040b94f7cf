"""Training with the global planner without a GPU (DESIGN.md §9x): the host twin of rlca_plan_shape against a float64
restatement (tests/planner_reward_ref.py) on oracle rollouts of stage 1, stage 2 and an arena map, the shaping's
properties on synthetic maps, every refusal (Planner, the trainer, the ABI, the command line) and the kernel's
resources."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import planner_reward_ref as rref
from helpers import random_actions
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.planner import HostState, Planner, build_plan_tables, fields_host, shape_host
from rl_collision_avoidance_b200.scenarios import arena_layout_host, arena_relayout_host, fill_config, make_scenario
from rl_collision_avoidance_b200.worldfile import WorldMap

F = np.float32
EPS = float(np.finfo(np.float32).eps)


def psi_bound(psi, w):
    """psi's bound against the float64 restatement: 8 ulp of |psi| + 2 |pose.w| + 1 (psi and the straight-line distance
    pose.w it subtracts, float32)"""
    return 8 * EPS * (abs(float(psi)) + 2.0 * abs(float(w)) + 1.0)


def shaped_bound(reward, term):
    """the shaped reward's bound against its float64 value from the same psi: 3 ulp of |reward| + |term|, term =
    gain (psi_prev - psi)"""
    return 3 * EPS * (abs(float(reward)) + abs(float(term)))


def _cfg(sc, W=1, auto_reset=0, seed=0):
    return fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512, auto_reset=auto_reset, seed=seed)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _oracle(sc, W, seed, auto_reset):
    from oracle.oracle import OracleWorld, OrcConfig
    ocfg = fill_config(OrcConfig(), sc, num_worlds=W, beams=512, auto_reset=auto_reset, seed=seed)
    return OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)


def _ticks(name, W, seed, ticks):
    """(sc, cfg, orc, generator): the generator yields after the run's start (flags None) and after every tick of an
    oracle rollout with random actions (arenas: parked robots and re-layouts as relayout_finished applies them)."""
    sc = make_scenario('arena', robots_per_world=8, arenas=4, arena_side=8.0, arena_seed=0) if name == 'arena' \
        else make_scenario(name)
    auto_reset = {'stage1': 1, 'stage2': 2, 'arena': 0}[name]
    cfg = _cfg(sc, W, auto_reset, seed)
    orc = _oracle(sc, W, seed, auto_reset)
    orc.reset_world()
    live = None
    if sc.layout is not None:
        orc.pose[:], orc.goal[:], orc.acc[:], status = arena_layout_host(cfg, sc.layout, orc.pose, orc.goal, orc.acc,
                                                                         pick=1)
        assert not status.any()
        orc.observe()
        live = np.ones(orc.N, np.uint8)
    else:
        orc.reset_pose()
    rng = np.random.default_rng(seed)

    def gen():
        nonlocal live
        yield None
        for _ in range(ticks):
            a = random_actions(rng, orc.N)
            a[:, 0] = np.abs(a[:, 0])
            orc.step(a, live)
            if sc.layout is not None:
                p, g, acc, meta, fl, live, status = arena_relayout_host(cfg, sc.layout, orc.pose, orc.goal, orc.acc,
                                                                        orc.meta, orc.flags, pick=1)
                assert not status.any()
                orc.pose[:], orc.goal[:], orc.acc[:], orc.meta[:], orc.flags[:] = p, g, acc, meta, fl
                orc.observe()
            yield orc.flags.copy()
    return sc, cfg, orc, gen()


@pytest.mark.parametrize('name, W, ticks', [('stage1', 2, 220), ('stage2', 1, 260), ('arena', 4, 300)])
def test_shape_twin_matches_float64_restatement(built, name, W, ticks):
    """psi of every row within 8 ulp of the float64 restatement (rows whose waypoint the restatement places
    differently, a segment through a cell corner, are skipped as test_planner allows); the shaped reward within 3 ulp of
    its float64 value on non-terminal ticks and the tick's bit for bit on terminal ones and where the goal is visible
    before and after; every written eplog return within float32 accumulation of the float64 sum of its episode's shaped
    rewards; psi_start and psi_prev reset on flags.w."""
    sc, cfg, orc, it = _ticks(name, W, 5, ticks)
    t = build_plan_tables(sc.map)
    m, N = sc.map, orc.N
    ppm, res, gain = float(F(cfg.ppm)), float(F(cfg.resolution)), float(F(cfg.progress_gain))
    hs = HostState(cfg, t)
    pp, ps = np.zeros(N, np.float32), np.zeros(N, np.float32)
    episode = [None] * N                  # per row: (tick rewards, flags, psis) of its running episode
    counts = dict(psi=0, shaped=0, kept=0, visible=0, returns=0, resets=0, skipped=0)
    for flags in it:
        fields_host(cfg, t, hs, orc.goal)
        reward, eplog = orc.reward.copy(), orc.eplog.copy()
        pp_before, ps_before, st_before = pp.copy(), ps.copy(), hs.status.copy()
        gs = orc.gs.copy()
        shape_host(cfg, t, hs, pp, ps, orc.pose, orc.goal, gs, flags, reward, eplog, in_place=True)
        for a in range(N):
            e = hs.entry[a]
            D, rect = (hs.row_field(a), tuple(hs.rect[a])) if e >= 0 else (None, None)
            s_ref, psi_ref = rref.psi(t.label, m.origin_cx, m.origin_cy, ppm, res, D, rect, e >= 0, orc.pose[a],
                                      orc.goal[a])
            if s_ref != hs.status[a]:
                counts['skipped'] += 1
            else:
                if abs(float(pp[a]) - psi_ref) > psi_bound(pp[a], orc.pose[a, 3]):
                    counts['skipped'] += 1          # another waypoint on the chain (a corner case of the walk)
                else:
                    counts['psi'] += 1
        if flags is None:
            assert np.array_equal(_bits(ps), _bits(pp))
            episode = [([], [], [float(pp[a])]) for a in range(N)]
            continue
        for a in range(N):
            fl = flags[a]
            if fl[0] == 0:
                want = rref.shaped_reward(orc.reward[a], fl, pp_before[a], pp[a], gain)
                tol = shaped_bound(orc.reward[a], gain * (float(pp_before[a]) - float(pp[a])))
                assert abs(float(reward[a]) - want) <= tol, (a, reward[a], want)
                counts['shaped'] += 1
                if st_before[a] == 0 and hs.status[a] == 0:
                    assert _bits(reward[a:a + 1]).tobytes() == _bits(orc.reward[a:a + 1]).tobytes()
                    counts['visible'] += 1
            else:
                assert _bits(reward[a:a + 1]).tobytes() == _bits(orc.reward[a:a + 1]).tobytes()
                counts['kept'] += 1
            ep = episode[a]
            if ep is not None:
                ep[0].append(float(orc.reward[a]))
                ep[1].append(fl.copy())
                ep[2].append(float(pp[a]))
            if fl[0] != 0 and fl[2] != 0:
                assert ep is not None
                want = rref.shaped_return(ep[0], ep[1], ep[2], gain)
                tol = 1e-6 * len(ep[0]) * (sum(abs(r) for r in ep[0]) + 1.0) + 1e-4
                assert abs(float(eplog[a, 2]) - want) <= tol, (a, eplog[a, 2], want, len(ep[0]))
                assert float(eplog[a, 2]) == float(F(F(orc.eplog[a, 2]) + F(F(gain) * F(ps_before[a] - pp_before[a]))))
                counts['returns'] += 1
                episode[a] = None
            if fl[3] != 0:
                assert ps[a] == pp[a]
                episode[a] = ([], [], [float(pp[a])])
                counts['resets'] += 1
            else:
                assert _bits(ps[a:a + 1]).tobytes() == _bits(ps_before[a:a + 1]).tobytes()
        # every other column of eplog is the tick's
        assert np.array_equal(_bits(np.delete(eplog, 2, 1)), _bits(np.delete(orc.eplog, 2, 1)))
    total = counts['psi'] + counts['skipped']
    assert counts['skipped'] <= max(2, total // 500), counts
    assert counts['shaped'] > 0 and counts['kept'] > 0 and counts['returns'] > 0 and counts['resets'] > 0, counts
    assert counts['visible'] > 0, counts


def _u_map():
    """A 0.2 m map, 12 m x 8 m, with a U-shaped wall open to the left: the goal inside the U, the robot behind it."""
    w, h = 60, 40
    c = np.zeros((h, w), np.uint8)
    c[0, :] = c[-1, :] = c[:, 0] = c[:, -1] = 254
    c[8:33, 35] = 254
    c[8, 20:36] = c[32, 20:36] = 254
    return WorldMap(cells=c, resolution=0.2, origin_cx=0, origin_cy=0, init_poses=np.zeros((0, 3)), name='U wall')


def test_detour_along_the_chain_earns_positive_shaped_progress(built):
    """A robot moved one descent-chain cell per tick round a U-shaped wall: on every tick that keeps status 1 and
    moves it away from the goal in straight-line terms, the shaped progress (tick progress plus psi_prev - psi) is
    positive."""
    import planner_ref as ref
    m = _u_map()
    sc = make_scenario('stage1', m, 1)
    cfg = _cfg(sc, 1)
    t = build_plan_tables(m)
    goal = np.array([[30 * 0.2 + 0.1, 20 * 0.2 + 0.1, 0.0, 0.0]], np.float32)
    pose = np.array([[45 * 0.2 + 0.1, 20 * 0.2 + 0.1, 0.0, 0.0]], np.float32)
    hs = HostState(cfg, t)
    fields_host(cfg, t, hs, goal)

    def dist(p):
        dx, dy = goal[0, 0] - p[0, 0], goal[0, 1] - p[0, 1]
        return F(np.sqrt(F(dx * dx + dy * dy)))

    pose[0, 3] = dist(pose)
    pp, ps = np.zeros(1, np.float32), np.zeros(1, np.float32)
    gs = np.zeros((1, 4), np.float32)
    shape_host(cfg, t, hs, pp, ps, pose, goal, gs, in_place=True)
    assert hs.status[0] == 1
    D, rect = hs.row_field(0), tuple(hs.rect[0])
    away = 0
    for _ in range(200):
        cx, cy = int(np.floor(pose[0, 0] * 5)), int(np.floor(pose[0, 1] * 5))
        if ref.field_at(D, rect, cx, cy) == 0:
            break
        nx, ny = ref.chain(D, rect, (cx, cy), 1)[0]
        st_prev, w_prev = hs.status[0], pose[0, 3]
        pose[0, 0], pose[0, 1] = F(nx * 0.2 + 0.1), F(ny * 0.2 + 0.1)
        pose[0, 3] = dist(pose)
        tick = F(cfg.progress_gain) * F(w_prev - pose[0, 3])
        reward = np.array([tick], np.float32)
        eplog = np.zeros((1, 8), np.float32)
        psi_prev = float(pp[0])
        shape_host(cfg, t, hs, pp, ps, pose, goal, gs, np.zeros((1, 4), np.uint8), reward, eplog, in_place=True)
        if st_prev == 1 and hs.status[0] == 1 and pose[0, 3] > w_prev:
            assert (float(w_prev) - float(pose[0, 3])) + (psi_prev - float(pp[0])) > 0
            assert reward[0] > 0
            away += 1
    assert away >= 10


# ---------------------------------------------------------------------------------------------- refusals
def test_planner_reward_needs_steer():
    with pytest.raises(ValueError, match='reward needs steer'):
        Planner(object(), steer=False, reward=True)


def test_trainer_refusals():
    from rl_collision_avoidance_b200.trainer import attach_planners
    with pytest.raises(ValueError, match='localization error needs a planner on the believed pose'):
        attach_planners([], 'geodesic', localization=object())
    with pytest.raises(ValueError, match="one of geodesic, straight, got 'bogus'"):
        attach_planners([], 'bogus')
    assert attach_planners([], None, localization=object()) is None


def test_trainer_refuses_the_circle_map_by_name():
    from rl_collision_avoidance_b200.trainer import attach_planners

    class _Env:
        sc = make_scenario('circle')

    class _Comp:
        env = _Env()
    with pytest.raises(ValueError, match=r'circle.*over the 58112-cell limit'):
        attach_planners([_Comp()], 'geodesic')


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'random', '--planner'], 'over the 58112-cell limit'),
    (['--mix', 'stage2:1,circle:1', '--planner'], '--planner on circle'),
    (['--scenario', 'arena', '--planner', '--pose-error', '0.1'], 'localization error needs a planner on the believed'),
    (['--scenario', 'arena', '--planner-reward', 'straight'], '--planner-reward needs --planner'),
    (['--scenario', 'arena', '--planner', '--planner-reward', 'euclid'], "invalid choice: 'euclid'"),
])
def test_cli_refusals(capsys, argv, message):
    import ppo_stage1
    from rl_collision_avoidance_b200.stage_world2 import StageWorld
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(stage=2, world_cls=StageWorld, num_env=44, batch_size=512, epoch=4, ckpt='stage2.pth',
                        argv=argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_abi_rejects_nulls(built):
    lib = _lib.load()
    sc = make_scenario('stage1')
    t = build_plan_tables(sc.map)
    cfg = _cfg(sc, 1)
    hs = HostState(cfg, t)
    z = lambda *s: np.zeros(s, np.float32)
    pose, goal, gs, out, pp, ps, rw = z(24, 4), z(24, 4), z(24, 4), z(24, 4), z(24), z(24), z(24)
    fl = np.zeros((24, 4), np.uint8)
    es = _lib.EnvState(pose.ctypes.data, goal.ctypes.data, None, None)
    T, S = C.byref(t.struct()), C.byref(hs.struct())
    p = lambda a: a.ctypes.data
    fields_host(cfg, t, hs, goal)
    assert lib.rlca_plan_shape_host(C.byref(cfg), T, S, p(pp), p(ps), C.byref(es), p(fl), p(rw), None, p(gs),
                                    p(gs)) == 0                                  # in place, no eplog
    assert lib.rlca_plan_shape_host(C.byref(cfg), T, S, None, p(ps), C.byref(es), None, None, None, p(gs), p(out)) == 1
    assert lib.rlca_plan_shape_host(C.byref(cfg), T, S, p(pp), None, C.byref(es), None, None, None, p(gs), p(out)) == 1
    assert lib.rlca_plan_shape_host(C.byref(cfg), T, S, p(pp), p(pp), C.byref(es), None, None, None, p(gs),
                                    p(out)) == 1                                 # psi_prev and psi_start alias
    assert lib.rlca_plan_shape_host(C.byref(cfg), T, S, p(pp), p(ps), C.byref(es), p(fl), None, None, p(gs),
                                    p(out)) == 1                                 # flags without reward
    assert lib.rlca_plan_shape_host(C.byref(cfg), T, S, p(pp), p(ps), None, None, None, None, p(gs), p(out)) == 1
    assert lib.rlca_plan_shape_host(C.byref(cfg), T, S, p(pp), p(ps), C.byref(es), None, None, None, None, p(out)) == 1
    assert lib.rlca_plan_shape_host(None, T, S, p(pp), p(ps), C.byref(es), None, None, None, p(gs), p(out)) == 1
    assert lib.rlca_plan_shape(C.byref(cfg), T, S, None, None, None, None, None, None, None, None, None) == 1
    with pytest.raises(ValueError, match='psi_prev must be a contiguous float32 array'):
        shape_host(cfg, t, hs, np.zeros(24), ps, pose, goal, gs)


def test_shape_kernel_resources(built, tmp_path):
    """-Xptxas -v on rlca_plan.cu: the shaping kernel keeps the waypoint kernel's budget, no spill, no stack, no shared
    memory."""
    import __graft_entry__ as g
    src = os.path.join(g.CSRC, 'rlca_plan.cu')
    r = subprocess.run([g.NVCC] + g.ARCH + g.COMMON + g.EXTRA['rlca_plan.cu'] +
                       ['-Xptxas', '-v', '-c', src, '-o', str(tmp_path / 'plan.o')], capture_output=True, text=True,
                       check=True)
    info = {}
    for m in re.finditer(r"Compiling entry function '(\w+)'.*?\n(.*?)Used (\d+) registers(.*?)\n", r.stderr, re.S):
        info[m.group(1)] = (m.group(2) + m.group(4), int(m.group(3)))
    shape = [k for k in info if 'rlca_plan_shape_kernel' in k]
    wp = [k for k in info if 'rlca_plan_waypoints_kernel' in k]
    assert shape and wp, r.stderr
    text, regs = info[shape[0]]
    assert '0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads' in text, text
    assert 'smem' not in text, text
    assert regs <= 64 and regs <= info[wp[0]][1] + 8, (regs, info[wp[0]][1])
