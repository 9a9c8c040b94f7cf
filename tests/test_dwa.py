"""The dynamic-window baseline without a GPU (DESIGN.md §9u): the float64 restatement (tests/dwa_ref.py) against a
brute-force sampling of the arcs, rlca_dwa_action_host against it on synthetic scans and on oracle states of stage 1,
stage 2 and the circle, the controller's properties, every argument check and command-line rule, and the kernel's
resources."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import dwa_ref
from helpers import make_pair, random_actions
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.evaluation import AUTO_RESET
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
CLEAR_TOL = 1e-4        # m, per-candidate clearance against float64
SCORE_TOL = 1e-5        # per-candidate score and the pick against the float64 best admissible score
MARGIN = 1e-4           # m: candidates this close to the admissibility boundary in float64 are excluded and counted;
                        # at most 1 % of them may be


def _cfg(scenario='stage1', worlds=1, beams=512):
    sc = make_scenario(scenario)
    return fill_config(_lib.EnvConfig(), sc, num_worlds=worlds, beams=beams, auto_reset=AUTO_RESET[scenario], seed=0)


def _scan_of_points(cfg, pts):
    """Normalised newest frame whose beams see the nearest of `pts` (robot frame) within half a beam's angle, the
    others no return."""
    from rl_collision_avoidance_b200.dwa import beam_directions
    b = np.arctan2(beam_directions(cfg)[:, 1], beam_directions(cfg)[:, 0]).astype(np.float64)
    r = np.full(len(b), float(cfg.range_max))
    half = (b[1] - b[0]) / 2
    for x, y in pts:
        a, d = math.atan2(y, x), math.hypot(x, y)
        j = np.flatnonzero(np.abs(b - a) <= half + 1e-12)
        r[j] = np.minimum(r[j], d)
    return (r / cfg.range_max - 0.5).astype(np.float32)


def _stack(frames):
    f = np.asarray(frames, np.float32)
    return np.ascontiguousarray(np.repeat(f[:, None, :], 3, 1))


def _check_against_ref(cfg, stack, gs, p):
    """Twin against float64 per robot; returns (excluded candidates, all candidates)."""
    from rl_collision_avoidance_b200.dwa import dwa_host
    act, status, clear, score = dwa_host(cfg, stack, gs, p, debug=True)
    cap = p.clearance_cap
    excluded = total = 0
    for a in range(len(gs)):
        ref = dwa_ref.robot(cfg, p, stack[a, 2], gs[a].astype(np.float64), cap)
        near = (np.abs(ref[:, 3]) < MARGIN) & (ref[:, 2] > 0)
        excluded += int(near.sum())
        total += len(ref)
        assert np.abs(clear[a] - ref[:, 2]).max() <= CLEAR_TOL, (a, np.abs(clear[a] - ref[:, 2]).max())
        assert np.abs(score[a] - ref[:, 4]).max() <= SCORE_TOL, (a, np.abs(score[a] - ref[:, 4]).max())
        adm = (ref[:, 2] > 0) & (ref[:, 3] >= 0)
        need = ref[:, 2] - ref[:, 3]
        np.testing.assert_array_equal(adm[~near], ((clear[a] > 0) & (clear[a] >= need))[~near])
        if (adm & ~near).any():
            assert status[a] == 0
            c = _index(cfg, p, gs[a], act[a])
            assert adm[c] or near[c], (a, c)
            best = ref[adm | near, 4].max()
            assert score[a][c] >= ref[adm & ~near, 4].max() - SCORE_TOL and score[a][c] <= best + SCORE_TOL
        elif not (adm | near).any():
            assert status[a] == 1 and act[a].tolist() == [0.0, 0.0]
    return excluded, total


def _index(cfg, p, gs, action):
    """Candidate index of the twin's pick (its (v, w) is one of the window's samples)."""
    vs, ws, _ = dwa_ref.window(cfg, p, float(gs[2]), float(gs[3]))
    d = np.abs(vs - action[0]) + np.abs(ws - action[1])
    return int(np.argmin(d))


# ---------------------------------------------------------------------------------------------- the reference itself
def test_reference_contact_against_sampling():
    """The closed-form contact arc length agrees with a float64 walk of the disc along the arc within its step, on
    straight lines, both turning directions, tight turns (R < rho) and points beside, ahead of and behind the path."""
    rng = np.random.default_rng(0)
    rho, step, length = 0.3, 2e-4, 2.5
    checked = hits = 0
    for v, w in [(1.0, 0.0), (1.0, 0.5), (1.0, -0.5), (0.5, 1.0), (0.1, -1.0), (0.8, 0.1), (0.2, 0.9)]:
        pts = rng.uniform(-2.5, 2.5, (400, 2))
        pts = pts[np.hypot(pts[:, 0], pts[:, 1]) >= rho]
        got = dwa_ref.contact(v, w, pts[:, 0], pts[:, 1], rho)
        for (x, y), g in zip(pts, got):
            want = dwa_ref.contact_sampled(v, w, x, y, rho, length, step)
            if math.isinf(want):
                assert g > length - step, (v, w, x, y, g)
            else:
                assert -1e-12 <= g - want + step <= step + 1e-9, (v, w, x, y, g, want)
                hits += 1
            checked += 1
    assert checked > 2000 and hits > 100, (checked, hits)


# ---------------------------------------------------------------------------------------------- twin vs float64
SYNTHETIC = ['empty', 'wall', 'cloud', 'within_rho', 'limits', 'beams180']


@pytest.mark.parametrize('case', SYNTHETIC)
def test_twin_matches_float64_synthetic(built, case):
    from rl_collision_avoidance_b200.dwa import DwaParams
    rng = np.random.default_rng(SYNTHETIC.index(case))
    cfg = _cfg('stage1', beams=180 if case == 'beams180' else 512)
    n = int(cfg.robots_per_world)
    frames, gs = [], []
    for i in range(n):
        if case == 'empty':
            pts = []
        elif case == 'wall':
            d = 0.5 + 0.1 * i
            pts = [(d, y) for y in np.linspace(-3, 3, 300)]
        elif case == 'within_rho':
            pts = [(0.2, 0.1)] + list(rng.uniform(-3, 3, (50, 2)))
        else:
            pts = list(rng.uniform(-3, 3, (rng.integers(20, 400), 2)))
        frames.append(_scan_of_points(cfg, pts))
        gs.append((rng.uniform(-8, 8), rng.uniform(-8, 8), rng.uniform(-0.2, 1.2), rng.uniform(-1.2, 1.2)))
    gs = np.asarray(gs, np.float32)
    p = DwaParams(accel=1.5, angular_accel=3.0) if case == 'limits' else DwaParams()
    excluded, total = _check_against_ref(cfg, _stack(frames), gs, p)
    assert excluded <= total // 100, (excluded, total)


@pytest.mark.parametrize('scenario,seed', [('stage1', 1), ('stage2', 2), ('circle', 3)])
def test_twin_matches_float64_oracle(built, scenario, seed):
    """Oracle states after 30 random-action ticks, the stack as the env's FIFO holds it."""
    from rl_collision_avoidance_b200.dwa import DwaParams
    sc, _, orc = make_pair(scenario, num_worlds=2, gpu=False, seed=seed, auto_reset=AUTO_RESET[scenario])
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(seed)
    stack = _stack(orc.obs)
    for _ in range(30):
        orc.step(random_actions(rng, orc.N))
        stack = np.ascontiguousarray(np.concatenate((stack[:, 1:], orc.obs[:, None, :]), 1))
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=2, beams=512, auto_reset=AUTO_RESET[scenario], seed=seed)
    for p in (DwaParams(), DwaParams(v_samples=7, w_samples=9, accel=2.0, angular_accel=4.0)):
        excluded, total = _check_against_ref(cfg, stack, orc.gs.copy(), p)
        assert excluded <= total // 100, (excluded, total)


# ---------------------------------------------------------------------------------------------- properties
def test_empty_scan_goal_ahead_drives_full_speed(built):
    from rl_collision_avoidance_b200.dwa import DwaParams, dwa_host
    cfg = _cfg()
    n = int(cfg.robots_per_world)
    stack = _stack([_scan_of_points(cfg, [])] * n)
    gs = np.tile(np.float32([5.0, 0.0, 0.3, 0.2]), (n, 1))
    act, status = dwa_host(cfg, stack, gs, DwaParams())
    assert (status == 0).all() and (act == np.float32([cfg.v_max, 0.0])).all(), act[:3]


def test_goal_behind_turns_towards_it(built):
    from rl_collision_avoidance_b200.dwa import DwaParams, dwa_host
    cfg = _cfg()
    n = int(cfg.robots_per_world)
    stack = _stack([_scan_of_points(cfg, [])] * n)
    left = np.tile(np.float32([-3.0, 0.5, 0.0, 0.0]), (n, 1))
    right = np.tile(np.float32([-3.0, -0.5, 0.0, 0.0]), (n, 1))
    a_l, _ = dwa_host(cfg, stack, left, DwaParams())
    a_r, _ = dwa_host(cfg, stack, right, DwaParams())
    assert (a_l[:, 1] > 0.5).all() and (a_r[:, 1] < -0.5).all(), (a_l[0], a_r[0])


def test_picks_are_admissible_and_inside_the_window(built):
    from rl_collision_avoidance_b200.dwa import DwaParams, dwa_host
    rng = np.random.default_rng(5)
    cfg = _cfg()
    n = int(cfg.robots_per_world)
    frames = [_scan_of_points(cfg, rng.uniform(-2, 2, (200, 2))) for _ in range(n)]
    gs = np.stack([rng.uniform(-6, 6, n), rng.uniform(-6, 6, n), rng.uniform(0, 1, n), rng.uniform(-1, 1, n)],
                  1).astype(np.float32)
    for p in (DwaParams(), DwaParams(accel=1.0, angular_accel=2.0)):
        act, status, clear, _ = dwa_host(cfg, _stack(frames), gs, p, debug=True)
        for a in np.flatnonzero(status == 0):
            c = _index(cfg, p, gs[a], act[a])
            v = np.float32(act[a, 0])
            need = v * np.float32(cfg.dt) + v * v / np.float32(2 * p.brake)
            assert clear[a, c] > 0 and clear[a, c] >= need, (a, clear[a, c], need)
            if p.accel:
                dv, dw = np.float32(p.accel * cfg.dt), np.float32(p.angular_accel * cfg.dt)
                assert gs[a, 2] - dv - 1e-6 <= act[a, 0] <= gs[a, 2] + dv + 1e-6
                assert gs[a, 3] - dw - 1e-6 <= act[a, 1] <= gs[a, 3] + dw + 1e-6
        for a in np.flatnonzero(status == 1):
            assert act[a].tolist() == [0.0, 0.0]


def test_return_within_rho_stops(built):
    from rl_collision_avoidance_b200.dwa import DwaParams, dwa_host
    cfg = _cfg()
    n = int(cfg.robots_per_world)
    stack = _stack([_scan_of_points(cfg, [(0.1, 0.25)])] * n)
    gs = np.tile(np.float32([5.0, 0.0, 0.5, 0.0]), (n, 1))
    act, status, clear, _ = dwa_host(cfg, stack, gs, DwaParams(), debug=True)
    assert (status == 1).all() and (act == 0).all() and (clear == 0).all()


def test_beam_directions_are_the_env_angles(built):
    """Identity at 512 beams; at 180 the env's nearest-index pick list, both ends exact."""
    from rl_collision_avoidance_b200.dwa import beam_directions
    for nb in (512, 180):
        cfg = _cfg(beams=nb)
        cs = beam_directions(cfg)
        assert cs.shape == (nb, 2) and cs.dtype == np.float32
        b = dwa_ref.beam_angles(cfg)
        np.testing.assert_array_equal(cs, np.stack((np.cos(b), np.sin(b)), 1).astype(np.float32))
        assert b[0] == -0.5 * float(cfg.fov) and abs(b[-1] - 0.5 * float(cfg.fov)) < 1e-12
    b = dwa_ref.beam_angles(_cfg(beams=512))
    np.testing.assert_allclose(np.diff(b), float(_cfg().fov) / 511, rtol=1e-9)


# ---------------------------------------------------------------------------------------------- argument rules
BAD = [(k, v) for k in ('radius', 'horizon', 'brake', 'clearance_cap') for v in (0.0, -1.0, math.nan, math.inf)] + \
    [(k, v) for k in ('heading_time', 'accel', 'angular_accel', 'heading_weight', 'clearance_weight', 'speed_weight')
     for v in (-0.1, math.nan, math.inf)] + \
    [('v_samples', 0), ('w_samples', 0), ('w_samples', 1025)]


@pytest.mark.parametrize('key,value', BAD)
def test_bad_parameters_raise(built, key, value):
    """DwaParams refuses the value, and so does the library's own check of the same struct, on both entries."""
    from rl_collision_avoidance_b200.dwa import DwaParams, beam_directions
    with pytest.raises(ValueError):
        DwaParams(**{key: value})
    cfg = _cfg()
    n = int(cfg.robots_per_world)
    ps = DwaParams().struct()
    setattr(ps, key, value)
    stack, gs = np.zeros((n, 3, 512), np.float32), np.zeros((n, 4), np.float32)
    act, status, cs = np.zeros((n, 2), np.float32), np.zeros(n, np.int32), beam_directions(cfg)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib = _lib.load()
    assert lib.rlca_dwa_action_host(C.byref(cfg), C.byref(ps), vp(cs), vp(stack), vp(gs), vp(act), vp(status), None,
                                    None) == 1
    assert lib.rlca_dwa_action(C.byref(cfg), C.byref(ps), vp(cs), vp(stack), vp(gs), vp(act), vp(status), None) == 1


def test_bad_buffers_and_configs_raise(built):
    from rl_collision_avoidance_b200.dwa import DwaParams, beam_directions
    cfg = _cfg()
    n = int(cfg.robots_per_world)
    ps = DwaParams().struct()
    stack, gs = np.zeros((n, 3, 512), np.float32), np.zeros((n, 4), np.float32)
    act, status, cs = np.zeros((n, 2), np.float32), np.zeros(n, np.int32), beam_directions(cfg)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib = _lib.load()
    args = [vp(cs), vp(stack), vp(gs), vp(act), vp(status)]
    assert lib.rlca_dwa_action_host(C.byref(cfg), C.byref(ps), *args, None, None) == 0
    for i in range(len(args)):
        bad = list(args)
        bad[i] = None
        assert lib.rlca_dwa_action_host(C.byref(cfg), C.byref(ps), *bad, None, None) == 1, i
        assert lib.rlca_dwa_action(C.byref(cfg), C.byref(ps), *bad, None) == 1, i
    assert lib.rlca_dwa_action_host(None, C.byref(ps), *args, None, None) == 1
    assert lib.rlca_dwa_action_host(C.byref(cfg), None, *args, None, None) == 1
    for field, value in (('beams', 1), ('beams', 513), ('v_max', 0.0), ('robots_per_world', 0), ('dt', 0.0)):
        bad = _cfg()
        setattr(bad, field, value)
        assert lib.rlca_dwa_action_host(C.byref(bad), C.byref(ps), *args, None, None) == 1, field
        assert lib.rlca_dwa_action(C.byref(bad), C.byref(ps), *args, None) == 1, field
    ps.v_samples, ps.w_samples = 32, 33
    assert lib.rlca_dwa_action_host(C.byref(cfg), C.byref(ps), *args, None, None) == 1


@pytest.mark.parametrize('argv, message', [
    (['--policy', os.path.join(CKPT, 'stage2.pth'), '--dwa-radius', '0.3'], '--dwa-radius applies to --baseline dwa only'),
    (['--baseline', 'nh-orca', '--dwa-samples', '5,5'], '--dwa-samples applies to --baseline dwa only'),
    (['--baseline', 'dwa', '--orca-map'], '--orca-map applies to --baseline orca / nh-orca only'),
    (['--baseline', 'dwa', '--orca-radius', '0.4'], '--orca-radius applies to --baseline orca / nh-orca only'),
    (['--baseline', 'dwa', '--nh-error', '0.2'], '--nh-error applies to --baseline orca / nh-orca only'),
    (['--baseline', 'dwa', '--hybrid'], '--hybrid applies to --policy only'),
    (['--baseline', 'dwa', '--dwa-samples', '5'], 'expected 2 comma-separated values'),
    (['--baseline', 'dwa', '--dwa-samples', '40,40'], 'at most 1024'),
    (['--baseline', 'dwa', '--dwa-weights', '1,-1,0'], 'clearance_weight must be finite and >= 0'),
    (['--baseline', 'dwa', '--dwa-accel', '1,2,3'], 'expected 1 to 2 comma-separated values'),
    (['--baseline', 'dwa', '--dwa-brake', '0'], 'brake must be finite and > 0'),
    (['--baseline', 'dwa', '--dwa-radius', 'nan'], 'radius must be finite and > 0'),
    (['--baseline', 'orca', '--scan-noise', '0.05'], 'the ORCA baselines do not read the scan'),
    (['--baseline', 'nh-orca', '--scan-delay', '2'], 'the ORCA baselines do not read the scan'),
    (['--baseline', 'orca', '--pose-error', '0.1'], 'the ORCA baselines and the hybrid driver read the true state'),
])
def test_evaluate_cli_rules(capsys, argv, message):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(['--scenario', 'stage2'] + argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_dwa_arguments_parse():
    import argparse

    from rl_collision_avoidance_b200 import dwa
    ap = argparse.ArgumentParser()
    ap.add_argument('--baseline')
    dwa.add_arguments(ap)
    args = ap.parse_args(['--baseline', 'dwa', '--dwa-samples', '5,7', '--dwa-accel', '1.5', '--dwa-weights', '2,0,1',
                          '--dwa-horizon', '3'])
    p = dwa.from_arguments(ap, args)
    assert (p.v_samples, p.w_samples, p.accel, p.angular_accel, p.horizon) == (5, 7, 1.5, 1.5, 3.0)
    assert (p.heading_weight, p.clearance_weight, p.speed_weight) == (2.0, 0.0, 1.0)
    assert dwa.from_arguments(ap, ap.parse_args(['--baseline', 'orca'])) is None


# ---------------------------------------------------------------------------------------------- resources
def test_kernel_uses_no_stack_or_local_memory(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_dwa.o')], check=True,
                         capture_output=True, text=True).stdout
    found = re.findall(r'Function \w*rlca_dwa_kernel\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', out)
    assert len(found) == 1, out
    reg, stack, shared, local = (int(x) for x in found[0])
    assert stack == 0 and local == 0 and reg <= 64, found
    assert shared <= 48 * 1024, found
