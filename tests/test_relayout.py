"""Training on random layouts without a GPU (DESIGN.md §9k): rlca_layout_respawn_host against a numpy restatement of the
parking and re-layout rule, its relation to rlca_layout_random_host, shard invariance, the failure status, every
rejected argument of rlca_layout_respawn / rlca_stack_refresh and of the trainers' and evaluate.py's command lines, and
the register budget of both kernels."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import layout_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario, random_layout_host, random_max_ticks, \
    relayout_host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
_F = np.float32


# ---------------------------------------------------------------------------------------------- numpy restatement
def _first_accept(seed, agent, episode, purpose, side, max_reject, ok_fn, chunk=64):
    for base in range(0, max_reject, chunk):
        ks = np.arange(base, min(base + chunk, max_reject))
        u = layout_ref.rand4(seed, agent, episode, ks, purpose)
        x = (u[0] - _F(0.5)) * _F(side)
        y = (u[1] - _F(0.5)) * _F(side)
        hit = np.flatnonzero(ok_fn(x, y))
        if len(hit):
            return x[hit[0]], y[hit[0]]
    return None


def _world_layout(seed, agent0, episode, R, side, sep2, tr2, max_reject):
    """(sx, sy, gx, gy, th) of one world at `episode`, or (1 + r) when robot r is not placed."""
    sx, sy, gx, gy = (np.zeros(0, _F) for _ in range(4))
    for r in range(R):
        a = (agent0 + r) & 0xFFFFFFFF
        s = _first_accept(seed, a, episode, 3, side, max_reject, lambda x, y: layout_ref._far(x, y, sx, sy, sep2))
        if s is None:
            return 1 + r
        x0, y0 = s
        sx, sy = np.append(sx, x0), np.append(sy, y0)
        g = _first_accept(seed, a, episode, 4, side, max_reject,
                          lambda x, y: layout_ref._far(x, y, _F([x0]), _F([y0]), tr2) & layout_ref._far(x, y, gx, gy,
                                                                                                           sep2))
        if g is None:
            return 1 + r
        gx, gy = np.append(gx, g[0]), np.append(gy, g[1])
    th = [layout_ref.normalize(layout_ref.rand4(seed, (agent0 + r) & 0xFFFFFFFF, episode, [0], 5)[0, 0] *
                               layout_ref.TWO_PI_F) for r in range(R)]
    return sx, sy, gx, gy, th


def relayout_ref(cfg, side, separation, min_travel, pose, goal, acc, meta, flags):
    """The rule of DESIGN.md §9k restated: latched robots parked, a world whose robots are all latched re-laid with the
    layout's draws at episode meta.y + 1 and its records written as a new episode."""
    R, W = int(cfg.robots_per_world), int(cfg.num_worlds)
    seed, mr = int(cfg.seed), int(cfg.max_reject)
    sep2, tr2 = _F(separation) * _F(separation), _F(min_travel) * _F(min_travel)
    pose, goal, acc = (np.array(a, _F, copy=True) for a in (pose, goal, acc))
    meta, flags = np.array(meta, np.int32, copy=True), np.array(flags, np.uint8, copy=True)
    live = np.zeros(R * W, np.uint8)
    status = np.zeros(W, np.int32)
    for w in range(W):
        rows = slice(w * R, (w + 1) * R)
        latched = meta[rows, 3] != 0
        if latched.all():
            e = int(meta[w * R, 1]) + 1
            agent0 = ((int(cfg.world_offset) + w) * R) & 0xFFFFFFFF
            lay = _world_layout(seed, agent0, e & 0xFFFFFFFF, R, side, sep2, tr2, mr)
            if isinstance(lay, tuple):
                sx, sy, gx, gy, th = lay
                for r in range(R):
                    i = w * R + r
                    pose[i, 0:3] = sx[r], sy[r], th[r]
                    if cfg.pre_distance_zero:
                        pose[i, 3] = 0.0
                    else:
                        ddx, ddy = _F(gx[r] - sx[r]), _F(gy[r] - sy[r])
                        pose[i, 3] = np.sqrt(layout_ref.fmaf(ddx, ddx, _F(ddy * ddy)))
                    goal[i] = gx[r], gy[r], 0.0, 0.0
                    acc[i, 0] = 0.0
                    acc[i, 2:4] = sx[r], sy[r]
                    meta[i, 0], meta[i, 1], meta[i, 3] = 1, e, 0
                    flags[i, 3] = 1
                live[rows] = 1
                continue
            status[w] = lay
        goal[w * R:(w + 1) * R][latched, 2:4] = 0.0
        live[rows] = (~latched).astype(np.uint8)
    return pose, goal, acc, meta, flags, live, status


# ---------------------------------------------------------------------------------------------- states
def _cfg(K, S, D, L, seed, W, world_offset=0, max_reject=4096, pre_zero=1, timeout=None):
    sc = make_scenario('random', robots_per_world=K, side=S, separation=D, min_travel=L, timeout=timeout)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512, seed=seed, world_offset=world_offset,
                      max_reject=max_reject)
    cfg.pre_distance_zero = pre_zero
    return sc, cfg


def _state(K, W, fill, kinds=('none', 'some', 'all')):
    """Rows of W worlds after a tick: world w latches none, some or all of its robots (kinds[w % len(kinds)]); the
    episode index meta.y is the same within a world, the stall flag and the tick's flags x..z are random."""
    rng = np.random.default_rng(fill)
    pose, goal, acc = (rng.standard_normal((K * W, 4)).astype(_F) for _ in range(3))
    meta = np.zeros((K * W, 4), np.int32)
    meta[:, 0] = rng.integers(1, 500, K * W)
    meta[:, 1] = np.repeat(rng.integers(1, 40, W), K)
    meta[:, 2] = rng.integers(0, 2, K * W)
    flags = rng.integers(0, 4, (K * W, 4)).astype(np.uint8)
    flags[:, 3] = 0
    for w in range(W):
        kind = kinds[w % len(kinds)]
        rows = slice(w * K, (w + 1) * K)
        if kind == 'all':
            meta[rows, 3] = 1
        elif kind == 'some':
            m = rng.integers(0, 2, K)
            m[0], m[-1] = 1, 0                          # at least one latched and one not
            meta[rows, 3] = rng.permutation(m)
    return pose, goal, acc, meta, flags


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


NAMES = ('pose', 'goal', 'acc', 'meta', 'flags', 'live', 'status')
# (K, S, D, L, seed, W, pre_distance_zero, max_reject)
REF_CASES = [(2, 10.0, 1.0, 5.0, 0, 9, 1, 4096), (8, 10.0, 1.0, 5.0, 3, 24, 1, 4096), (8, 10.0, 1.0, 5.0, 4, 12, 0, 4096),
             (16, 10.0, 1.0, 5.0, 5, 12, 1, 4096), (32, 10.0, 1.0, 5.0, 6, 6, 1, 4096),
             (64, 20.0, 1.0, 10.0, 1, 3, 0, 4096), (16, 8.0, 1.0, 4.0, 0, 24, 1, 8)]


@pytest.mark.parametrize('K,S,D,L,seed,W,pre_zero,max_reject', REF_CASES)
def test_host_equals_numpy_restatement(built, K, S, D, L, seed, W, pre_zero, max_reject):
    sc, cfg = _cfg(K, S, D, L, seed, W, max_reject=max_reject, pre_zero=pre_zero)
    rows = _state(K, W, seed)
    got = relayout_host(cfg, sc.layout, *rows)
    want = relayout_ref(cfg, S, D, L, *rows)
    for name, x, y in zip(NAMES, got, want):
        assert _bits_equal(x, y), name
    relaid = got[4][:, 3].reshape(W, K).all(1)
    assert relaid.any()
    if max_reject == 8:                                  # some all-latched worlds are re-laid and some fail
        assert got[6].any() and (relaid | (got[6] != 0)).sum() > got[6].astype(bool).sum()


def test_parking_and_new_episode_records(built):
    K, W = 8, 30
    sc, cfg = _cfg(K, 10.0, 1.0, 5.0, 2, W)
    pose, goal, acc, meta, flags = rows = _state(K, W, 7)
    p2, g2, a2, m2, f2, live, status = relayout_host(cfg, sc.layout, *rows)
    assert not status.any()
    latched = meta[:, 3] != 0
    world_all = latched.reshape(W, K).all(1)
    relaid = np.repeat(world_all, K)
    parked = latched & ~relaid
    # parking: the last command is zero and live is 0 exactly for the latched robots of worlds not re-laid
    assert not g2[parked, 2:4].any() and (live[parked] == 0).all()
    assert (live[~parked] == 1).all()
    untouched = ~relaid
    assert _bits_equal(g2[untouched & ~latched], goal[untouched & ~latched])
    assert _bits_equal(g2[parked, 0:2], goal[parked, 0:2])
    for x, y in ((p2, pose), (a2, acc), (m2, meta), (f2, flags)):
        assert _bits_equal(x[untouched], y[untouched])
    # was_reset only on re-laid robots; their new episode
    assert np.array_equal(f2[:, 3] != 0, relaid)
    assert _bits_equal(f2[:, 0:3], flags[:, 0:3])
    assert (m2[relaid, 0] == 1).all() and (m2[relaid, 3] == 0).all()
    assert np.array_equal(m2[relaid, 1], meta[relaid, 1] + 1)
    assert np.array_equal(m2[relaid, 2], meta[relaid, 2])                  # the stall flag is kept
    assert not a2[relaid, 0].any() and _bits_equal(a2[relaid, 1], acc[relaid, 1])
    assert _bits_equal(a2[relaid, 2:4], p2[relaid, 0:2]) and not g2[relaid, 2:4].any()
    assert not p2[relaid, 3].any()                                        # pre_distance_zero


def test_episode_zero_is_the_layout_of_rlca_layout_random(built):
    """meta.y = -1 in every world, all robots latched: the re-layout draws episode 0 and equals the evaluation layout
    of rlca_layout_random_host - one sampler, not two."""
    for K, S, W, pre_zero in ((8, 10.0, 40, 1), (64, 20.0, 3, 0), (3, 6.0, 17, 1)):
        sc, cfg = _cfg(K, S, 1.0, 0.5 * S, 5, W, pre_zero=pre_zero)
        pose, goal, acc, meta, flags = _state(K, W, 3, kinds=('all',))
        meta[:, 1] = -1
        got = relayout_host(cfg, sc.layout, pose, goal, acc, meta, flags)
        want = random_layout_host(cfg, sc.layout, pose, goal, acc)
        assert not want[3].any() and not got[6].any()
        assert _bits_equal(got[0], want[0]) and _bits_equal(got[1][:, 0:2], want[1][:, 0:2])
        assert _bits_equal(got[2][:, 1:4], want[2][:, 1:4])
        assert (got[3][:, 1] == 0).all()


def test_layouts_differ_between_episodes(built):
    K, W = 8, 16
    sc, cfg = _cfg(K, 10.0, 1.0, 5.0, 1, W)
    pose, goal, acc, meta, flags = _state(K, W, 1, kinds=('all',))
    meta[:, 1] = 1
    first = relayout_host(cfg, sc.layout, pose, goal, acc, meta, flags)
    meta[:, 1] = 2
    second = relayout_host(cfg, sc.layout, pose, goal, acc, meta, flags)
    assert not np.any(np.all(first[0][:, 0:2] == second[0][:, 0:2], axis=1))


def test_world_rows_do_not_depend_on_num_worlds_or_sharding(built):
    K, W = 8, 60
    sc, cfg = _cfg(K, 10.0, 1.0, 5.0, 2, W)
    rows = _state(K, W, 9)
    one = relayout_host(cfg, sc.layout, *rows)
    parts = []
    for w0, wc in ((0, 25), (25, 35)):
        _, c = _cfg(K, 10.0, 1.0, 5.0, 2, wc, world_offset=w0)
        parts.append(relayout_host(c, sc.layout, *(r[w0 * K:(w0 + wc) * K] for r in rows)))
    for i, name in enumerate(NAMES):
        assert _bits_equal(np.concatenate([q[i] for q in parts]), one[i]), name


def test_failed_world_keeps_its_rows_and_stays_parked(built):
    """K = 64 in a 6 m square: every world fails at the robot the restatement names, keeps its rows with the last
    command zeroed, and stays latched (the next call fails the same way)."""
    K, W = 64, 2
    sc, cfg = _cfg(K, 6.0, 1.0, 3.0, 0, W)
    rows = _state(K, W, 0, kinds=('all',))
    got = relayout_host(cfg, sc.layout, *rows)
    want = relayout_ref(cfg, 6.0, 1.0, 3.0, *rows)
    assert got[6].all() and np.array_equal(got[6], want[6])
    assert not got[5].any() and not got[4][:, 3].any()
    for x, y in zip(got[:5], (rows[0], rows[1], rows[2], rows[3], rows[4])):
        if x is got[1]:
            assert _bits_equal(x[:, 0:2], y[:, 0:2]) and not x[:, 2:4].any()
        else:
            assert _bits_equal(x, y)
    again = relayout_host(cfg, sc.layout, *got[:5])
    assert np.array_equal(again[6], got[6])


# ---------------------------------------------------------------------------------------------- rejections
def test_abi_rejects_bad_arguments(built):
    lib = _lib.load()
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    K, W = 8, 2
    sc, cfg = _cfg(K, 10.0, 1.0, 5.0, 0, W)
    pose, goal, acc, meta, flags = _state(K, W, 0)
    live, status = np.zeros(K * W, np.uint8), np.zeros(W, np.int32)
    good = _lib.LayoutParams(10.0, 1.0, 5.0)
    bufs = [vp(pose), vp(goal), vp(acc), vp(meta), vp(flags), vp(live), vp(status)]
    host = lambda c, prm, *b: lib.rlca_layout_respawn_host(c, prm, *b)
    assert host(C.byref(cfg), C.byref(good), *bufs) == 0
    for i in range(len(bufs)):
        bad = list(bufs)
        bad[i] = None
        assert host(C.byref(cfg), C.byref(good), *bad) == 1, i
    assert host(None, C.byref(good), *bufs) == 1
    assert host(C.byref(cfg), None, *bufs) == 1
    nan, inf = float('nan'), float('inf')
    bad_params = [(0.0, 1.0, 0.0), (nan, 1.0, 0.0), (10.0, 1.0, -0.01), (10.0, 1.0, 14.15), (10.0, 0.5, 5.0),
                  (10.0, nan, 5.0), (10.0, inf, 5.0)]
    for prm in bad_params:
        assert host(C.byref(cfg), C.byref(_lib.LayoutParams(*prm)), *bufs) == 1, prm
    bad_cfgs = []
    for field, value in (('robots_per_world', 1), ('robots_per_world', 65), ('num_worlds', 0), ('max_reject', 0),
                         ('world_offset', -1), ('auto_reset', 1), ('auto_reset', 2)):
        c = _lib.EnvConfig.from_buffer_copy(cfg)
        setattr(c, field, value)
        bad_cfgs.append(c)
        assert host(C.byref(c), C.byref(good), *bufs) == 1, (field, value)
    # the device entry checks its arguments before it launches anything
    state = _lib.EnvState(vp(pose), vp(goal), vp(acc), vp(meta))
    dev = lambda c, prm, s, f, lv, st: lib.rlca_layout_respawn(c, prm, s, f, lv, st, None)
    dbufs = [vp(flags), vp(live), vp(status)]
    assert dev(None, C.byref(good), C.byref(state), *dbufs) == 1
    assert dev(C.byref(cfg), None, C.byref(state), *dbufs) == 1
    assert dev(C.byref(cfg), C.byref(good), None, *dbufs) == 1
    for i in range(3):
        bad = list(dbufs)
        bad[i] = None
        assert dev(C.byref(cfg), C.byref(good), C.byref(state), *bad) == 1, i
    for field in ('pose_dev', 'goal_dev', 'acc_dev', 'meta_dev'):
        s2 = _lib.EnvState(vp(pose), vp(goal), vp(acc), vp(meta))
        setattr(s2, field, None)
        assert dev(C.byref(cfg), C.byref(good), C.byref(s2), *dbufs) == 1, field
    for prm in bad_params:
        assert dev(C.byref(cfg), C.byref(_lib.LayoutParams(*prm)), C.byref(state), *dbufs) == 1, prm
    for c in bad_cfgs:
        assert dev(C.byref(c), C.byref(good), C.byref(state), *dbufs) == 1
    assert b'auto_reset must be 0' in lib.rlca_last_error()


def test_stack_refresh_rejects_bad_arguments(built):
    lib = _lib.load()
    _, cfg = _cfg(8, 10.0, 1.0, 5.0, 0, 2)
    p = [C.c_void_p(0x10000 * (k + 1)) for k in range(5)]       # aligned, never dereferenced: every call fails first
    call = lambda c, *b: lib.rlca_stack_refresh(c, *b, None)
    for i in range(5):
        bad = list(p)
        bad[i] = None
        assert call(C.byref(cfg), *bad) == 1, i
    assert call(None, *p) == 1
    for i in range(1, 5):                                        # flags are bytes; the others must be 16-byte aligned
        bad = list(p)
        bad[i] = C.c_void_p(p[i].value + 4)
        assert call(C.byref(cfg), *bad) == 1, i
        assert b'misaligned' in lib.rlca_last_error()
    for field, value in (('beams', 2), ('beams', 0), ('beams', 511), ('robots_per_world', 0), ('num_worlds', 0),
                         ('robots_per_world', 65)):
        c = _lib.EnvConfig.from_buffer_copy(cfg)
        setattr(c, field, value)
        assert call(C.byref(c), *p) == 1, (field, value)


def test_make_scenario_random_timeout():
    assert make_scenario('random').timeout == 10000
    assert make_scenario('random', timeout=426).timeout == 426
    assert random_max_ticks(10.0) == 426
    for bad in (0, -3, 2.5, 2 ** 31):
        with pytest.raises(ValueError, match='timeout must be an integer >= 1'):
            make_scenario('random', timeout=bad)
    for name in ('stage1', 'stage2', 'circle'):
        with pytest.raises(ValueError, match='shape the random scenario only'):
            make_scenario(name, timeout=100)


def _trainer(stage):
    import ppo_stage1
    if stage == 1:
        return lambda argv: ppo_stage1.main(argv=argv)
    import ppo_stage2
    return lambda argv: ppo_stage1.main(stage=2, world_cls=None, num_env=ppo_stage2.NUM_ENV,
                                        batch_size=ppo_stage2.BATCH_SIZE, epoch=ppo_stage2.EPOCH, ckpt='stage2.pth',
                                        argv=argv)


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'random'], '--scenario random trains with ppo_stage2.py'),
    (['--scenario', 'random', '--random-robots', '16'], '--scenario random trains with ppo_stage2.py'),
    (['--random-robots', '8'], 'apply to --scenario random only'),
])
def test_stage1_cli_rejects_random(capsys, argv, message):
    with pytest.raises(SystemExit) as e:
        _trainer(1)(argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


@pytest.mark.parametrize('argv, message', [
    (['--random-robots', '8'], '--random-min-travel / --random-timeout apply to --scenario random only'),
    (['--scenario', 'stage2', '--random-timeout', '100'], 'apply to --scenario random only'),
    (['--scenario', 'circle', '--random-side', '8'], 'apply to --scenario random only'),
    (['--scenario', 'random', '--random-robots', '1'], 'robots_per_world must be in 2..64'),
    (['--scenario', 'random', '--random-robots', '65'], 'robots_per_world must be in 2..64'),
    (['--scenario', 'random', '--random-side', '0'], 'side must be finite and > 0'),
    (['--scenario', 'random', '--random-side', '70'], 'is not on free cells of the map'),
    (['--scenario', 'random', '--random-separation', '0.5'], 'separation must be finite and >'),
    (['--scenario', 'random', '--random-min-travel', '15'], 'min_travel must be in'),
    (['--scenario', 'random', '--random-timeout', '0'], '--random-timeout must be >= 1'),
    (['--scenario', 'random', '--random-timeout', '-5'], '--random-timeout must be >= 1'),
])
def test_stage2_cli_rejects_bad_random(capsys, argv, message):
    with pytest.raises(SystemExit) as e:
        _trainer(2)(argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'random', '--random-timeout', '100'], 'unrecognized arguments: --random-timeout'),
    (['--scenario', 'circle', '--random-robots', '8'],
     '--random-robots / --random-side / --random-separation / --random-min-travel apply to --scenario random only'),
])
def test_evaluate_cli_has_no_training_flags(capsys, argv, message):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(argv + ['--policy', os.path.join(CKPT, 'stage2.pth')])
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_kernels_do_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_layout.o')], check=True,
                         capture_output=True, text=True).stdout
    for name in ('rlca_layout_respawn_kernel', 'rlca_stack_refresh_kernel'):
        m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % name, out)
        assert m, (name, out)
        assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
        assert int(m.group(1)) <= 64, m.group(0)


def test_random_timeout_defaults():
    """A trainer's random episode times out after random_max_ticks(S) unless --random-timeout says otherwise;
    evaluate.py's random scenario keeps make_scenario's 10000."""
    import argparse
    from rl_collision_avoidance_b200.scenarios import add_random_arguments, random_scenario_from_arguments
    for timeout_flag, argv, want in ((True, [], 426), (True, ['--random-side', '20'], random_max_ticks(20.0)),
                                     (True, ['--random-timeout', '50'], 50), (False, [], 10000)):
        ap = argparse.ArgumentParser()
        ap.add_argument('--scenario', default='random')
        add_random_arguments(ap, timeout=timeout_flag)
        assert random_scenario_from_arguments(ap, ap.parse_args(argv)).timeout == want, argv
