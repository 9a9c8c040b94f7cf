"""The arena curriculum without a GPU (DESIGN.md §9z): the update twin and the weighted layout and re-layout twins
against a numpy restatement of the rule (tests/curriculum_ref.py), equal weights against pick 1's twins, the draw
frequencies, the fused tally, every refusal (ABI, ArenaCurriculum, its state and the command lines), the kernels'
resources and the per-arena grouping of evaluation partials."""
import ctypes as C
import math
import os
import re
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
from scipy import stats

import curriculum_ref
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.curriculum import ArenaCurriculum, CurriculumParams, check_params, layout_host, \
    relayout_host, update_host
from rl_collision_avoidance_b200.scenarios import arena_layout_host, arena_relayout_host, arena_tables_struct, \
    fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
_F = np.float32


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype.itemsize == b.dtype.itemsize and np.array_equal(a.view(np.uint8),
                                                                                          b.view(np.uint8))


def _setup(K, T, seed, W, world_offset=0, max_reject=4096, pre_zero=1, fill=0, side=10.0, obstacles=(4, 10), D=None,
           L=None):
    sc = make_scenario('arena', robots_per_world=K, arenas=T, arena_side=side, obstacles=obstacles, separation=D,
                       min_travel=L, pick=1)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512, seed=seed, world_offset=world_offset,
                      max_reject=max_reject)
    cfg.pre_distance_zero = pre_zero
    rng = np.random.default_rng(fill)
    rows = tuple(rng.standard_normal((K * W, 4)).astype(_F) for _ in range(3))
    return sc, cfg, rows


def _equal_cdf(T, w):
    return (np.arange(T + 1, dtype=np.uint64) * np.uint64(w)).astype(np.uint64)


def _random_cdf(T, rng):
    w = rng.integers(1, 1 << 20, T, endpoint=True).astype(np.uint64)
    w[rng.integers(0, T)] = 1
    cdf = np.zeros(T + 1, np.uint64)
    cdf[1:] = np.cumsum(w)
    return cdf


# ---------------------------------------------------------------------------------------------- the update
@pytest.mark.parametrize('T', [1, 7, 64, 576])
@pytest.mark.parametrize('decay,uniform', [(0.0, 0.0), (0.9, 0.1), (float(np.nextafter(_F(1), _F(0))), 1.0),
                                           (0.5, 0.0), (0.0, 1.0)])
def test_update_twin_equals_restatement(built, T, decay, uniform):
    rng = np.random.default_rng(T)
    for _ in range(3):
        E = (rng.random(T) * 500).astype(_F)
        S = (E * rng.random(T)).astype(_F)
        S[::5] = 0
        S[1::5] = E[1::5]
        pending = np.concatenate([rng.integers(0, 400, T), np.zeros(T, np.int64)]).astype(np.int32)
        pending[T:] = (pending[:T] * rng.random(T)).astype(np.int32)
        got = update_host(E, S, pending, decay, uniform)
        want = curriculum_ref.fold(E, S, pending, decay, uniform)
        assert _bits_equal(got[0], want[0]) and _bits_equal(got[1], want[1])
        assert not got[2].any()
        assert np.array_equal(got[3], want[3]) and got[3][0] == 0


def test_equal_counts_give_equal_weights_never_below_one(built):
    T = 40
    # the start: E = S = 0, p = 1/2, every weight 2^20
    _, _, _, cdf = update_host(np.zeros(T, _F), np.zeros(T, _F), np.zeros(2 * T, np.int32), 0.9, 0.1)
    assert np.array_equal(cdf, _equal_cdf(T, 1 << 20))
    for e, s in ((100.0, 50.0), (1e6, 0.0), (1e6, 1e6), (3.0, 1.0)):
        _, _, _, cdf = update_host(np.full(T, e, _F), np.full(T, s, _F), np.zeros(2 * T, np.int32), 0.5, 0.0)
        w = np.diff(cdf)
        assert (w == w[0]).all() and w[0] >= 1, (e, s)
    # always solved or never solved with no uniform share: the weight floor 1
    _, _, _, cdf = update_host(np.array([1e7, 1e7, 0], _F), np.array([0, 1e7, 0], _F), np.zeros(6, np.int32), 0.5,
                               0.0)
    assert list(np.diff(cdf)) == [1, 1, 1 << 20]


def test_decay_pulls_a_stale_arena_back_to_one_half(built):
    """An arena solved every time that gets no new episodes scores higher at every update, towards p = 1/2."""
    E, S = np.array([200, 200], _F), np.array([200, 100], _F)
    last = 0
    for _ in range(50):
        E, S, _, cdf = update_host(E, S, np.zeros(4, np.int32), 0.8, 0.1)
        w = np.diff(cdf)
        assert w[0] >= last
        last = w[0]
    assert w[0] > 0.99 * (1 << 20)


# ---------------------------------------------------------------------------------------------- equal weights: pick 1
# (K, T, seed, W, world_offset, pre_distance_zero, max_reject)
LAYOUT_CASES = [(2, 4, 0, 6, 0, 1, 4096), (8, 64, 4, 12, 0, 0, 4096), (16, 9, 1, 10, 5, 1, 4096),
                (24, 16, 7, 5, 100, 1, 4096), (12, 2, 0, 3, 0, 1, 8)]


@pytest.mark.parametrize('K,T,seed,W,wo,pre_zero,max_reject', LAYOUT_CASES)
@pytest.mark.parametrize('weight', [1, 977, 1 << 20])
def test_equal_weights_lay_out_as_pick_1(built, K, T, seed, W, wo, pre_zero, max_reject, weight):
    small = max_reject == 8
    sc, cfg, rows = _setup(K, T, seed, W, wo, max_reject, pre_zero, side=5.0 if small else 10.0,
                           obstacles=(0, 0) if small else (4, 10), D=1.2 if small else None, L=1.0 if small else None)
    got = layout_host(cfg, sc.layout, _equal_cdf(T, weight), np.full(W, -3), *rows)
    want = arena_layout_host(cfg, sc.layout, *rows, pick=1)
    for x, y in zip(got[:4], want):
        assert _bits_equal(x, y)
    assert bool(want[3].any()) == small
    assert ((got[4] == -3) == (want[3] != 0)).all()


def _state(K, W, fill):
    """Rows after a tick: world w latches none, some or all of its robots (w mod 3); flags with every outcome."""
    rng = np.random.default_rng(fill)
    pose, goal, acc = (rng.standard_normal((K * W, 4)).astype(_F) for _ in range(3))
    meta = np.zeros((K * W, 4), np.int32)
    meta[:, 0] = rng.integers(1, 500, K * W)
    meta[:, 1] = np.repeat(rng.integers(1, 40, W), K)
    meta[:, 2] = rng.integers(0, 2, K * W)
    flags = rng.integers(0, 4, (K * W, 4)).astype(np.uint8)
    flags[:, 3] = 0
    for w in range(W):
        rows = slice(w * K, (w + 1) * K)
        if w % 3 == 2:
            meta[rows, 3] = 1
        elif w % 3 == 1:
            m = rng.integers(0, 2, K)
            m[0], m[-1] = 1, 0
            meta[rows, 3] = rng.permutation(m)
    return pose, goal, acc, meta, flags


# (K, T, seed, W, pre_distance_zero, max_reject)
RELAYOUT_CASES = [(8, 64, 3, 24, 1, 4096), (8, 9, 4, 12, 0, 4096), (16, 16, 5, 12, 1, 4096), (10, 4, 0, 24, 1, 8)]


@pytest.mark.parametrize('K,T,seed,W,pre_zero,max_reject', RELAYOUT_CASES)
def test_equal_weights_relay_as_pick_1(built, K, T, seed, W, pre_zero, max_reject):
    sc, cfg, _ = _setup(K, T, seed, W, max_reject=max_reject, pre_zero=pre_zero)
    rows = _state(K, W, seed)
    wa = np.arange(W, dtype=np.int32) % T
    got = relayout_host(cfg, sc.layout, _equal_cdf(T, 1 << 20), wa, np.zeros(2 * T, np.int32), None, *rows)
    want = arena_relayout_host(cfg, sc.layout, *rows, pick=1)
    for name, x, y in zip(('pose', 'goal', 'acc', 'meta', 'flags', 'live', 'status'), got, want):
        assert _bits_equal(x, y), name
    if max_reject == 8:
        assert want[6].any()
    relaid = want[4][:, 3].reshape(W, K).all(1)
    assert relaid.any()
    assert np.array_equal(got[7][~relaid], wa[~relaid])


# ---------------------------------------------------------------------------------------------- unequal weights
@pytest.mark.parametrize('K,T,seed,W,wo,pre_zero,max_reject', LAYOUT_CASES)
def test_weighted_layout_equals_restatement(built, K, T, seed, W, wo, pre_zero, max_reject):
    small = max_reject == 8
    sc, cfg, rows = _setup(K, T, seed, W, wo, max_reject, pre_zero, side=5.0 if small else 10.0,
                           obstacles=(0, 0) if small else (4, 10), D=1.2 if small else None, L=1.0 if small else None)
    cdf = _random_cdf(T, np.random.default_rng(seed))
    wa = np.full(W, -1, np.int32)
    got = layout_host(cfg, sc.layout, cdf, wa, *rows)
    want = curriculum_ref.layout(cfg, sc.layout, cdf, wa, *rows)
    for name, x, y in zip(('pose', 'goal', 'acc', 'status', 'world_arena'), got, want):
        assert _bits_equal(x, y), name


@pytest.mark.parametrize('K,T,seed,W,pre_zero,max_reject', RELAYOUT_CASES)
@pytest.mark.parametrize('masked', [False, True])
def test_weighted_relayout_equals_restatement(built, K, T, seed, W, pre_zero, max_reject, masked):
    sc, cfg, _ = _setup(K, T, seed, W, max_reject=max_reject, pre_zero=pre_zero)
    rows = _state(K, W, seed)
    rng = np.random.default_rng(seed + 1)
    cdf = _random_cdf(T, rng)
    wa = rng.integers(0, T, W).astype(np.int32)
    pending = rng.integers(0, 9, 2 * T).astype(np.int32)
    mask = (rng.random(K * W) < 0.3).astype(np.uint8) if masked else None
    got = relayout_host(cfg, sc.layout, cdf, wa, pending, mask, *rows)
    want = curriculum_ref.relayout(cfg, sc.layout, cdf, wa, pending, mask, *rows)
    for name, x, y in zip(('pose', 'goal', 'acc', 'meta', 'flags', 'live', 'status', 'world_arena', 'pending'), got,
                          want):
        assert _bits_equal(x, y), name


def test_layouts_cover_the_multi_round_path(built):
    """At least one accepted try past the first 32-try round in the cases above (arena_ref's restatement)."""
    import arena_ref
    most = 0
    for K, T, seed, W, wo, pre_zero, max_reject in LAYOUT_CASES[:4]:
        sc, cfg, rows = _setup(K, T, seed, W, wo, max_reject, pre_zero)
        most = max(most, int(arena_ref.layout(cfg, sc.layout, 1, *rows)[5].max()))
    assert most >= 32, most


def test_draws_follow_the_weights(built):
    """Arena frequencies over 6000 worlds' layouts (K = 2, 8 arenas) follow w / sum(w): chi-square p > 1e-4."""
    T, W = 8, 6000
    sc, cfg, rows = _setup(2, T, 21, W, obstacles=(0, 2))
    w = np.array([1 << 20, 1 << 18, 1 << 19, 40000, 1 << 20, 300000, 1 << 17, 700000], np.uint64)
    cdf = np.zeros(T + 1, np.uint64)
    cdf[1:] = np.cumsum(w)
    _, _, _, status, wa = layout_host(cfg, sc.layout, cdf, np.full(W, -1), *rows)
    assert not status.any()
    counts = np.bincount(wa, minlength=T)
    expected = w.astype(np.float64) / float(w.sum()) * W
    assert stats.chisquare(counts, expected).pvalue > 1e-4, (counts, expected)


def test_tally_counts_ended_unmasked_rows_against_the_old_arena(built):
    """Every world latched and re-laid: the pending counts are the tick's ended rows (x != 0, z != 0; z == 1 a success)
    of the unmasked robots, added to the arena each world held before, while world_arena moves on."""
    K, T, W = 6, 5, 40
    sc, cfg, _ = _setup(K, T, 2, W)
    pose, goal, acc, meta, flags = _state(K, W, 9)
    meta[:, 3] = 1
    rng = np.random.default_rng(4)
    flags[:, 0] = rng.integers(0, 2, K * W)
    flags[:, 2] = rng.integers(0, 4, K * W)
    mask = np.tile(np.array([1, 0, 0, 1, 0, 0], np.uint8), W)
    wa = rng.integers(0, T, W).astype(np.int32)
    cdf = _random_cdf(T, rng)
    got = relayout_host(cfg, sc.layout, cdf, wa, np.zeros(2 * T, np.int32), mask, pose, goal, acc, meta, flags)
    ended = (flags[:, 0] != 0) & (flags[:, 2] != 0) & (mask == 0)
    ok = ended & (flags[:, 2] == 1)
    want = np.zeros(2 * T, np.int64)
    for w in range(W):
        want[wa[w]] += ended[w * K:(w + 1) * K].sum()
        want[T + wa[w]] += ok[w * K:(w + 1) * K].sum()
    assert np.array_equal(got[8], want) and want[:T].sum() > 0
    assert not got[6].any() and not np.array_equal(got[7], wa)
    unmasked = relayout_host(cfg, sc.layout, cdf, wa, np.zeros(2 * T, np.int32), None, pose, goal, acc, meta, flags)
    assert unmasked[8][:T].sum() == ((flags[:, 0] != 0) & (flags[:, 2] != 0)).sum()


def test_weighted_layout_is_shard_invariant(built):
    sc, cfg, rows = _setup(8, 16, 2, 120)
    cdf = _random_cdf(16, np.random.default_rng(3))
    big = layout_host(cfg, sc.layout, cdf, np.zeros(120), *rows)
    parts = []
    for w0, wc in ((0, 3), (3, 67), (70, 50)):
        c = fill_config(_lib.EnvConfig(), sc, num_worlds=wc, beams=512, seed=2, world_offset=w0)
        parts.append(layout_host(c, sc.layout, cdf, np.zeros(wc), *(r[w0 * 8:(w0 + wc) * 8] for r in rows)))
    for i in range(5):
        assert _bits_equal(np.concatenate([q[i] for q in parts]), big[i]), i


# ---------------------------------------------------------------------------------------------- refusals
def test_abi_rejects_bad_arguments(built):
    lib = _lib.load()
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    K, T, W = 8, 4, 2
    sc, cfg, (p, g, a) = _setup(K, T, 0, W)
    t = sc.layout.tables
    tab = arena_tables_struct(t)
    good = _lib.LayoutParams(0.0, 1.2, 5.0)
    cdf, wa, pend = _equal_cdf(T, 5), np.zeros(W, np.int32), np.zeros(2 * T, np.int32)
    E, S = np.zeros(T, _F), np.zeros(T, _F)
    bufs = [cdf, wa, pend, E, S]
    cur = _lib.ArenaCurriculum(T, *(vp(b) for b in bufs))
    st = np.zeros(W, np.int32)
    lay = lambda c, prm, tb, cu: lib.rlca_layout_arena_weighted_host(c, prm, tb, cu, vp(p), vp(g), vp(a), vp(st))
    assert lay(C.byref(cfg), C.byref(good), C.byref(tab), C.byref(cur)) == 0
    bad_curs = [None]
    for i in range(5):
        ptrs = [vp(b) for b in bufs]
        ptrs[i] = None
        bad_curs.append(C.byref(_lib.ArenaCurriculum(T, *ptrs)))
    bad_curs.append(C.byref(_lib.ArenaCurriculum(T + 1, *(vp(b) for b in bufs))))      # not the tables' T
    bad_curs.append(C.byref(_lib.ArenaCurriculum(0, *(vp(b) for b in bufs))))
    for cu in bad_curs:
        assert lay(C.byref(cfg), C.byref(good), C.byref(tab), cu) == 1
    # check_arena's refusals
    assert lay(None, C.byref(good), C.byref(tab), C.byref(cur)) == 1
    assert lay(C.byref(cfg), None, C.byref(tab), C.byref(cur)) == 1
    assert lay(C.byref(cfg), C.byref(good), None, C.byref(cur)) == 1
    assert lay(C.byref(cfg), C.byref(_lib.LayoutParams(0.0, 1.0, 5.0)), C.byref(tab), C.byref(cur)) == 1
    empty = t.cell_off.copy()
    empty[2] = empty[1]
    assert lay(C.byref(cfg), C.byref(good), C.byref(_lib.ArenaTables(T, empty.ctypes.data, t.cells.ctypes.data)),
               C.byref(cur)) == 1
    for field, v in (('num_worlds', 0), ('max_reject', 0), ('world_offset', -1), ('robots_per_world', 65)):
        c = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512)
        setattr(c, field, v)
        assert lay(C.byref(c), C.byref(good), C.byref(tab), C.byref(cur)) == 1, field
    # T >= 2^20 on tables of as many arenas
    big = 1 << 20
    boff = np.arange(big + 1, dtype=np.int32)
    bcells = np.zeros(big, np.int32)
    btab = _lib.ArenaTables(big, boff.ctypes.data, bcells.ctypes.data)
    bcur = _lib.ArenaCurriculum(big, *(vp(b) for b in bufs))
    assert lay(C.byref(cfg), C.byref(good), C.byref(btab), C.byref(bcur)) == 1
    assert 'num_arenas must be in [1, 2^20)' in lib.rlca_last_error().decode()
    # the re-layout twin: the same, auto_reset 0, and no NULL buffer but the row mask
    meta, flags, live = np.zeros((K * W, 4), np.int32), np.zeros((K * W, 4), np.uint8), np.zeros(K * W, np.uint8)
    rb = [vp(p), vp(g), vp(a), vp(meta), vp(flags), vp(live), vp(st)]
    rel = lambda c, cu, mask, *b: lib.rlca_layout_arena_weighted_respawn_host(c, C.byref(good), C.byref(tab), cu, mask,
                                                                              *b)
    assert rel(C.byref(cfg), C.byref(cur), None, *rb) == 0
    for i in range(len(rb)):
        bad = list(rb)
        bad[i] = None
        assert rel(C.byref(cfg), C.byref(cur), None, *bad) == 1, i
    for cu in bad_curs:
        assert rel(C.byref(cfg), cu, None, *rb) == 1
    c = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=512, auto_reset=True)
    assert rel(C.byref(c), C.byref(cur), None, *rb) == 1
    # the update
    upd = lambda cu, d, u: lib.rlca_arena_curriculum_update_host(cu, d, u)
    assert upd(C.byref(cur), 0.9, 0.1) == 0 and upd(C.byref(cur), 0.0, 1.0) == 0
    for d, u in ((1.0, 0.1), (-0.1, 0.1), (math.nan, 0.1), (math.inf, 0.1), (0.9, -0.01), (0.9, 1.01),
                 (0.9, math.nan)):
        assert upd(C.byref(cur), d, u) == 1, (d, u)
    for cu in bad_curs[:6] + [C.byref(_lib.ArenaCurriculum(0, *(vp(b) for b in bufs))), C.byref(bcur)]:
        assert upd(cu, 0.9, 0.1) == 1
    # the device entries check their arguments before they launch anything
    state = _lib.EnvState(vp(p), vp(g), vp(a), vp(meta))
    dev = lambda c, tb, cu, s, status: lib.rlca_layout_arena_weighted(c, C.byref(good), tb, cu, s, status, None)
    assert dev(C.byref(cfg), C.byref(tab), None, C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(tab), bad_curs[-2], C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), None, C.byref(cur), C.byref(state), vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(tab), C.byref(cur), None, vp(st)) == 1
    assert dev(C.byref(cfg), C.byref(tab), C.byref(cur), C.byref(state), None) == 1
    rdev = lambda c, cu, s: lib.rlca_layout_arena_weighted_respawn(c, C.byref(good), C.byref(tab), cu, None, s,
                                                                   vp(flags), vp(live), vp(st), None)
    assert rdev(C.byref(c), C.byref(cur), C.byref(state)) == 1                     # auto_reset 1
    assert rdev(C.byref(cfg), bad_curs[3], C.byref(state)) == 1                    # pending NULL
    assert rdev(C.byref(cfg), C.byref(cur), C.byref(_lib.EnvState(vp(p), vp(g), vp(a), None))) == 1
    assert lib.rlca_arena_curriculum_update(C.byref(cur), 1.0, 0.1, None) == 1
    assert lib.rlca_arena_curriculum_update(bad_curs[1], 0.9, 0.1, None) == 1


@pytest.mark.parametrize('decay,uniform,message', [(1.0, 0.1, 'decay must be in [0, 1)'),
                                                   (-0.5, 0.1, 'decay must be in [0, 1)'),
                                                   (math.nan, 0.1, 'decay must be in [0, 1)'),
                                                   (0.9, 1.5, 'uniform must be in [0, 1]'),
                                                   (0.9, math.nan, 'uniform must be in [0, 1]')])
def test_params_rejected(decay, uniform, message):
    with pytest.raises(ValueError, match=re.escape(message)):
        check_params(CurriculumParams(decay, uniform))


def test_curriculum_rejects_other_scenarios():
    """ArenaCurriculum refuses before it touches the device: another scenario, or arenas with pick 0."""
    for sc, message in ((make_scenario('random'), 'needs an arena scenario, got random'),
                        (make_scenario('arena', arenas=4, pick=0), 'the scenario has pick 0')):
        with pytest.raises(ValueError, match=re.escape(message)):
            ArenaCurriculum(SimpleNamespace(sc=sc), CurriculumParams())
    with pytest.raises(ValueError, match='decay must be in'):
        ArenaCurriculum(SimpleNamespace(sc=make_scenario('arena', arenas=4, pick=1)), CurriculumParams(1.0, 0.1))


def test_load_state_dict_rejects_other_arenas():
    import torch
    cur = ArenaCurriculum.__new__(ArenaCurriculum)          # the state checks need no device buffers
    cur.T, cur.arena_seed = 4, 0
    for name in ('E', 'S'):
        setattr(cur, name, torch.zeros(4))
    cur.cdf, cur.pending = torch.zeros(5, dtype=torch.int64), torch.zeros(8, dtype=torch.int32)
    sd = {'num_arenas': 4, 'arena_seed': 0, 'E': torch.ones(4), 'S': torch.ones(4),
          'cdf': torch.arange(5, dtype=torch.int64), 'pending': torch.zeros(8, dtype=torch.int32)}
    cur.load_state_dict(sd)
    assert torch.equal(cur.cdf, torch.arange(5)) and torch.equal(cur.E, torch.ones(4))
    for change, message in ((dict(num_arenas=5), 'holds 5 arenas, the scenario has 4'),
                            (dict(arena_seed=1), 'is for arena seed 1, the scenario has 0'),
                            (dict(E=torch.ones(3)), 'E is (3,)'),
                            (dict(cdf=torch.arange(5, dtype=torch.int32)), 'cdf is (5,) torch.int32')):
        with pytest.raises(ValueError, match=re.escape(message)):
            cur.load_state_dict(dict(sd, **change))


@pytest.mark.parametrize('argv, message', [
    (['--scenario', 'stage2', '--arena-curriculum'], '--arena-curriculum needs --scenario arena or an arena component'),
    (['--scenario', 'random', '--arena-curriculum'], '--arena-curriculum needs --scenario arena'),
    (['--mix', 'stage2:2,random:3', '--arena-curriculum'], '--arena-curriculum needs --scenario arena'),
    (['--scenario', 'arena', '--arena-count', '4', '--arena-curriculum', '--curriculum-decay', '1'],
     'decay must be in [0, 1)'),
    (['--scenario', 'arena', '--arena-count', '4', '--arena-curriculum', '--curriculum-decay', 'nan'],
     'decay must be in [0, 1)'),
    (['--scenario', 'arena', '--arena-count', '4', '--arena-curriculum', '--curriculum-uniform', '-0.1'],
     'uniform must be in [0, 1]'),
    (['--scenario', 'arena', '--arena-count', '4', '--curriculum-decay', '0.5'],
     '--curriculum-decay / --curriculum-uniform apply with --arena-curriculum only'),
])
def test_stage2_cli_rejects_bad_curriculum(capsys, argv, message):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(stage=2, argv=argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_stage1_cli_rejects_curriculum(capsys):
    import ppo_stage1
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(stage=1, argv=['--arena-curriculum'])
    assert e.value.code == 2
    assert '--arena-curriculum needs --scenario arena' in capsys.readouterr().err


def test_evaluate_cli_rejects_per_arena_off_arenas(capsys):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(['--scenario', 'random', '--per-arena', '--policy', os.path.join(CKPT, 'stage2.pth')])
    assert e.value.code == 2
    assert '--per-arena applies to --scenario arena only' in capsys.readouterr().err


# ---------------------------------------------------------------------------------------------- resources
def test_kernels_do_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_layout.o')], check=True,
                         capture_output=True, text=True).stdout
    for name in ('rlca_layout_arena_weighted_kernel', 'rlca_layout_arena_weighted_respawn_kernel',
                 'rlca_arena_curriculum_update_kernel'):
        m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % name, out)
        assert m, (name, out)
        assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
        assert int(m.group(1)) <= 64, m.group(0)


# ---------------------------------------------------------------------------------------------- per-arena evaluation
def test_per_arena_sums_to_the_totals():
    from rl_collision_avoidance_b200.evaluation import NPARTIALS, metrics, per_arena, totals
    T, W, wo = 7, 30, 12
    lay = SimpleNamespace(count=T, tables=SimpleNamespace(cell_off=np.cumsum([0] + list(range(5, 5 + T)))))
    rng = np.random.default_rng(0)
    p = rng.random((W, NPARTIALS)) * 10
    p[:, :4] = rng.integers(0, 9, (W, 4))
    rows = per_arena(p, lay, wo)
    assert [r['arena'] for r in rows] == list(range(T)) and [r['cells'] for r in rows] == list(range(5, 5 + T))
    assert sum(r['worlds'] for r in rows) == W
    assert np.allclose(sum(r['totals'] for r in rows), totals(p), rtol=1e-12, atol=0)
    for k in ('episodes', 'reached', 'crashed', 'timed_out', 'unfinished'):
        assert sum(r['metrics'][k] for r in rows) == metrics(totals(p))[k], k
    a3 = [w for w in range(W) if (wo + w) % T == 3]
    assert np.array_equal(rows[3]['totals'], totals(p[a3]))
