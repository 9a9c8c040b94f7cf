"""Safety metrics without a GPU (DESIGN.md §9m): the host twins of csrc/rlca_safety.cu against hand-computed
separations, the numpy restatement (tests/safety_ref.py) and a float64 brute force; the contact bound on oracle
rollouts; the per-episode fold on a scripted sequence; the reduction; every rejected argument; the kernel's
registers."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import safety_ref
from helpers import make_pair, random_actions
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.evaluation import SAFETY_COLUMNS, safety_contact, safety_reduce_host, \
    safety_separation_host, safety_totals, safety_track_host
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario, random_layout_host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
_F = np.float32
INF = _F(np.inf)


def _cfg(R=2, W=1, scenario='circle', beams=8, auto_reset=0):
    sc = make_scenario(scenario)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=beams, auto_reset=auto_reset)
    cfg.robots_per_world = R
    return cfg


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _sep(cfg, a, b):
    return safety_separation_host(cfg, np.atleast_2d(_F(a)), np.atleast_2d(_F(b)))


# ------------------------------------------------------------------------------------------------ separation
def test_column_names_follow_the_header(built):
    src = open(os.path.join(ROOT, 'include', 'rlca.h')).read()
    idx = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r'#define RLCA_SAFETY_([A-Z_]+) (\d+)', src)}
    assert idx.pop('npartials') == len(SAFETY_COLUMNS) == len(safety_ref.COLUMNS)
    for name, i in idx.items():
        assert SAFETY_COLUMNS[i] == name, (name, i)
    assert SAFETY_COLUMNS == safety_ref.COLUMNS


def test_separation_hand_cases(built):
    cfg = _cfg()
    cfg.half_len, cfg.half_wid = 0.25, 0.125                       # exactly representable extents
    hl, hw = 0.25, 0.125
    # side by side along x, gap 0.5; along y, gap 0.25
    assert _sep(cfg, (0, 0, 0), (1.0, 0, 0))[0] == _F(0.5)
    assert _sep(cfg, (0, 0, 0), (0, 0.5, 0))[0] == _F(0.25)
    # corner to corner: offsets (2 hl + 0.3, 2 hw + 0.4) -> 0.5
    assert abs(float(_sep(cfg, (0, 0, 0), (2 * hl + 0.3, 2 * hw + 0.4, 0))[0]) - 0.5) < 1e-6
    # corner to edge at 45 degrees: B's corner points at A's right edge; its tip is r_c from B's centre
    th = math.pi / 4 + math.atan2(hw, hl)                          # a corner of B on the -x axis of B's centre
    r_c = math.hypot(hl, hw)
    got = float(_sep(cfg, (0, 0, 0), (hl + 0.3 + r_c, 0, math.pi - math.atan2(hw, hl)))[0])
    assert abs(got - 0.3) < 1e-6, (got, th)
    # overlapping, touching inside, crossed
    assert _sep(cfg, (0, 0, 0), (0.3, 0.1, 0.4))[0] == 0.0
    assert _sep(cfg, (0, 0, 0), (0, 0, math.pi / 2))[0] == 0.0
    # within reach of the edge only: B above A's top edge, shifted, both corners of B's bottom edge beyond A's corners
    cfg.half_len = 1.0
    long_ = _sep(cfg, (0, 0, 0), (0.25, 0.75, math.pi / 2))[0]      # B upright: half extents (0.125, 1.0) -> bottom at -0.25
    assert long_ == 0.0
    got = _sep(cfg, (0, 0, 0), (0.25, 1.5, math.pi / 2))[0]         # B's bottom edge at y = 0.5, A's top at 0.125
    assert abs(float(got) - 0.375) < 1e-6


def test_separation_is_symmetric_and_equals_the_restatement(built):
    cfg = _cfg()
    rng = np.random.default_rng(0)
    n = 10000
    a = np.zeros((n, 4), np.float32)
    b = np.zeros((n, 4), np.float32)
    a[:, 0:2] = rng.uniform(-20, 20, (n, 2))
    a[:, 2] = rng.uniform(-np.pi, np.pi, n)
    b[:, 0:2] = a[:, 0:2] + rng.uniform(-1.5, 1.5, (n, 2)) * (rng.random((n, 1)) < 0.8) \
        + rng.uniform(-12, 12, (n, 2)) * (rng.random((n, 1)) < 0.3)
    b[:, 2] = rng.uniform(-np.pi, np.pi, n)
    a[:50, 2] = b[:50, 2] = 0.0                                    # parallel edges
    got = safety_separation_host(cfg, a, b)
    assert _bits_equal(got, safety_separation_host(cfg, b, a))
    want = safety_ref.separation(safety_ref.corners(a, cfg.half_len, cfg.half_wid),
                                 safety_ref.corners(b, cfg.half_len, cfg.half_wid))
    assert _bits_equal(got, want), np.nonzero(got != want)[0][:8]
    assert (got == 0).sum() > 500 and (got > 0).sum() > 5000
    # float64 brute force over densely sampled outlines: s <= sampled minimum <= s + step (and a rounding margin)
    m = 2000
    CA = safety_ref.corners(a[:m], cfg.half_len, cfg.half_wid).astype(np.float64)
    CB = safety_ref.corners(b[:m], cfg.half_len, cfg.half_wid).astype(np.float64)
    per_edge = 64
    step = 2 * max(cfg.half_len, cfg.half_wid) / per_edge
    t = np.arange(per_edge)[None, None, :, None] / per_edge
    outline = lambda Cn: (Cn[:, :, None, :] * (1 - t) + np.roll(Cn, -1, 1)[:, :, None, :] * t).reshape(len(Cn), -1, 2)
    PA, PB = outline(CA), outline(CB)
    for lo in range(0, m, 100):
        d = np.linalg.norm(PA[lo:lo + 100, :, None, :] - PB[lo:lo + 100, None, :, :], axis=3).min(axis=(1, 2))
        s = got[lo:lo + 100].astype(np.float64)
        assert (s <= d + 1e-5).all() and (d <= s + step + 1e-5).all(), (np.abs(d - s).max(), step)


def test_contact_bound_value(built):
    cfg = _cfg()
    got = safety_contact(cfg)
    assert got.view(np.uint32) == safety_ref.contact(cfg).view(np.uint32)
    r_c = math.hypot(cfg.half_len, cfg.half_wid)
    want = math.sqrt(2) * cfg.resolution + 2 * cfg.dt * (cfg.v_max + max(abs(cfg.w_min), abs(cfg.w_max)) * r_c)
    assert abs(float(got) - want) < 1e-6


# ------------------------------------------------------------------------------------------------ oracle rollouts
class _Host:
    """rlca_safety_track_host next to a host copy of the episode tracker's boundaries."""

    def __init__(self, cfg, episodes, near_dist=0.1):
        self.cfg, self.E, self.near_dist = cfg, episodes, near_dist
        N = cfg.robots_per_world * cfg.num_worlds
        self.closed = np.full(N, -1, np.int32)
        self.count = np.zeros(N, np.int32)
        self.results = np.zeros((N, episodes, 4), np.float32)
        self.state = dict(min_sep=np.full(N, INF, np.float32), min_clear=np.full(N, INF, np.float32),
                          last_clear=np.full(N, INF, np.float32), near=np.zeros(N, np.int32),
                          partner=np.full(N, -1, np.int32), records=np.zeros((N, episodes, 4), np.float32))

    def tick(self, pose_in, meta_in, pose_out, flags, obs):
        safety_track_host(self.cfg, self.near_dist, pose_in, meta_in, pose_out, flags, obs, self.closed, self.count,
                          self.state)
        for a in np.nonzero((self.closed != meta_in[:, 1]) & (flags[:, 2] != 0))[0]:      # the episode tracker's rule
            if self.count[a] < self.E:
                self.results[a, self.count[a], 0] = flags[a, 2]
            self.count[a] += 1
            self.closed[a] = meta_in[a, 1]


def _env_cfg(orc):
    cfg = _lib.EnvConfig()
    for name, _ in cfg._fields_:
        setattr(cfg, name, getattr(orc.cfg, name))
    return cfg


def _rollout(orc, host, ticks, actions, ref=None):
    for t in range(ticks):
        pose_in, meta_in = orc.pose.copy(), orc.meta.copy()
        orc.step(actions(t))
        host.tick(pose_in, meta_in, orc.pose, orc.flags, orc.obs)
        if ref is not None:
            ref.tick(pose_in, meta_in, orc.pose, orc.flags, orc.obs)


def _causes(host):
    """(cause, both-in-range, hit, result) of every record."""
    out = []
    for a in range(len(host.count)):
        for i in range(min(int(host.count[a]), host.E)):
            packed = int(host.state['records'][a, i, 3])
            out.append((packed & 3, bool(packed & 4), ((packed >> 8) & 0xff) - 1, int(host.results[a, i, 0]), a))
    return out


def test_two_robots_head_on_is_a_robot_crash(built):
    """Two robots on a 1.5 m circle drive at each other over free floor: cause robot, each charged to the other."""
    sc, _, orc = make_pair('circle', num_worlds=1, beams=64, auto_reset=0, gpu=False, robots_per_world=2, radius=1.5)
    orc.reset_world()
    orc.reset_pose()
    host = _Host(_env_cfg(orc), 1)
    ref = safety_ref.Tracker(host.cfg, 1, 0.1)
    act = np.float32([[1.0, 0.0], [1.0, 0.0]])
    _rollout(orc, host, 40, lambda t: act, ref)
    causes = _causes(host)
    assert len(causes) == 2 and all(c[3] == 2 for c in causes), causes
    assert [(c[0], c[2]) for c in causes] == [(2, 1), (2, 0)]
    rec = host.state['records'][:, 0]
    assert (rec[:, 0] <= safety_contact(host.cfg)).all() and (rec[:, 0] > 0).all()    # stopped before they overlap
    for k, v in ref.state().items():
        assert _bits_equal(host.state[k], v), k


def test_one_robot_into_a_wall_is_a_static_crash(built):
    """Single-robot stage-1 worlds under random forward actions: every crash is static, R = 1 gives +inf separation."""
    sc, _, orc = make_pair('stage1', num_worlds=48, beams=64, auto_reset=1, gpu=False, robots_per_world=1, seed=3)
    orc.reset_world()
    orc.reset_pose()
    host = _Host(_env_cfg(orc), 6)
    rng = np.random.default_rng(4)
    _rollout(orc, host, 300, lambda t: random_actions(rng, orc.N))
    causes = _causes(host)
    crashes = [c for c in causes if c[3] == 2]
    assert len(crashes) >= 5, len(crashes)
    assert all(c[0] == 1 and c[2] == -1 for c in crashes)
    assert all(c[0] == 0 for c in causes if c[3] != 2)
    n = np.minimum(host.count, host.E)
    rec = np.concatenate([host.state['records'][a, :n[a]] for a in range(orc.N)])
    assert np.isinf(rec[:, 0]).all() and (rec[:, 2] == 0).all()
    assert (rec[:, 3].astype(np.int64) >> 16 == 0).all()


def test_every_crash_on_free_floor_is_a_robot_crash(built):
    """Random layouts in a 5 m square far from any wall, random actions: the contact bound never calls a crash static,
    and the host twin equals the restatement bit for bit along the way."""
    K, W = 8, 24
    sc = make_scenario('random', robots_per_world=K, side=5.0, separation=0.8, min_travel=2.0)
    from oracle.oracle import OracleWorld, OrcConfig
    ocfg = fill_config(OrcConfig(), sc, num_worlds=W, beams=64, auto_reset=0, seed=7)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    orc.reset_world()
    orc.reset_pose()
    cfg = _env_cfg(orc)
    pose, goal, acc, status = random_layout_host(cfg, sc.layout, orc.pose, orc.goal, orc.acc)
    assert not status.any()
    orc.pose[:], orc.goal[:], orc.acc[:] = pose, goal, acc
    orc.observe()
    host = _Host(cfg, 1)
    ref = safety_ref.Tracker(cfg, 1, 0.1)
    rng = np.random.default_rng(8)
    _rollout(orc, host, 120, lambda t: random_actions(rng, orc.N), ref)
    crashes = [c for c in _causes(host) if c[3] == 2]
    assert len(crashes) >= 20, len(crashes)
    assert all(c[0] == 2 and 0 <= c[2] < K and c[2] != c[4] % K for c in crashes), crashes[:4]
    for k, v in ref.state().items():
        assert _bits_equal(host.state[k], v), k
    assert np.array_equal(host.count, ref.count) and np.array_equal(host.closed, ref.closed)


# ------------------------------------------------------------------------------------------------ scripted fold
def _scripted(cfg, host, ref, steps):
    """steps: (pose_in, ep_in, pose_out, flags) per tick with (R, 3) poses; obs from `clear` metres."""
    for pose_in, ep, pose_out, flags, clear in steps:
        R = len(pose_in)
        pi = np.zeros((R, 4), np.float32)
        po = np.zeros((R, 4), np.float32)
        pi[:, :3], po[:, :3] = pose_in, pose_out
        meta = np.zeros((R, 4), np.int32)
        meta[:, 1] = ep
        obs = np.full((R, cfg.beams), 0.5, np.float32)
        obs[:, 3] = _F(clear) / _F(cfg.range_max) - _F(0.5)
        fl = np.asarray(flags, np.uint8)
        host.tick(pi, meta, po, fl, obs)
        ref.tick(pi, meta, po, fl, obs)


def test_fold_on_a_scripted_sequence(built):
    cfg = _cfg(R=2, W=1, beams=8, auto_reset=1)
    cfg.half_len, cfg.half_wid = 0.25, 0.125
    E, near = 2, 0.25
    host, ref = _Host(cfg, E, near), safety_ref.Tracker(cfg, E, near)
    far = lambda gap: [(0, 0, 0), (0.5 + gap, 0, 0)]               # side by side, footprints `gap` apart
    none, reach, crash_respawn = (0, 0, 0, 0), (1, 0, 1, 0), (1, 1, 2, 1)
    steps = [
        # near_dist exactly is not a near miss; just below is
        (far(1.0), [0, 0], far(0.25), [none, none], [3.0, 2.0]),
        (far(0.25), [0, 0], far(0.125), [none, none], [1.0, 2.5]),
        # robot 0 crashes and is re-spawned far away in the tick: its separation is taken at the poses the tick started
        # from (0.125), not at its new pose; its scan (0.1 m, at the new pose) is not the ended episode's
        (far(0.125), [0, 0], [(9, 9, 0), (0.5 + 0.125, 0, 0)], [crash_respawn, none], [0.1, 2.0]),
        # episode 1 of robot 0; robot 1 reaches its goal and is not re-spawned (auto_reset 0 / 2 behaviour)
        ([(9, 9, 0), (0.625, 0, 0)], [1, 0], [(9, 9, 0), (0.625, 0, 0)], [none, reach], [4.0, 1.5]),
        # robot 1 idles latched: nothing is tracked for it, whatever comes close
        ([(9, 9, 0), (0.625, 0, 0)], [1, 0], [(1.0, 0, 0), (0.625, 0, 0)], [none, (1, 0, 0, 0)], [0.3, 0.2]),
        # robot 0 ends episode 1 and later a third episode: the third is counted and dropped (E = 2)
        ([(1.0, 0, 0), (0.625, 0, 0)], [1, 0], [(1.0, 0, 0), (0.625, 0, 0)], [(1, 0, 3, 1), (1, 0, 0, 0)], [0.3, 0.2]),
        ([(5, 5, 0), (0.625, 0, 0)], [2, 0], [(5, 5, 0), (0.625, 0, 0)], [(1, 0, 1, 1), (1, 0, 0, 0)], [0.3, 0.2]),
    ]
    _scripted(cfg, host, ref, steps)
    for k, v in ref.state().items():
        assert _bits_equal(host.state[k], v), k
    rec = host.state['records']
    bound = float(safety_contact(cfg))
    assert 0.125 <= bound
    # robot 0, episode 0: min separation 0.125 to robot 1, near-miss ticks 2 and 3 (0.25 on tick 1 is not below 0.25)
    assert rec[0, 0, 0] == _F(0.125) and abs(rec[0, 0, 1] - 1.0) < 1e-5 and rec[0, 0, 2] == 2.0
    assert int(rec[0, 0, 3]) == (2 | 2 << 8 | 2 << 16)             # robot, charged to robot 1, partner robot 1
    # robot 0, episode 1: poses (9, 9) then (1, 0): the footprints overlap robot 1's at the end -> 0
    assert rec[0, 1, 0] == 0.0 and abs(rec[0, 1, 1] - 0.3) < 1e-5 and int(rec[0, 1, 3]) == (0 | 2 << 16)
    assert host.count[0] == 3 and host.count[1] == 1
    # robot 1: one record, reached, min separation 0.125 on tick 2 (on tick 3 robot 0 already stands at its new pose),
    # scans 2.0, 2.5, 2.0, 1.5
    assert rec[1, 0, 0] == _F(0.125) and abs(rec[1, 0, 1] - 1.5) < 1e-5 and rec[1, 0, 2] == 1.0
    assert int(rec[1, 0, 3]) == (0 | 1 << 16) and not rec[1, 1].any()
    # the running state is reset after an end
    assert np.isinf(host.state['min_sep']).all() and (host.state['partner'] == -1).all()
    assert abs(host.state['last_clear'][0] - 0.3) < 1e-5


def test_both_in_range_uses_the_previous_scan(built):
    cfg = _cfg(R=2, W=1, beams=8, auto_reset=1)
    cfg.half_len, cfg.half_wid = 0.25, 0.125
    crash = (1, 1, 2, 1)
    for prev_clear, flag in ((0.05, 4), (3.0, 0)):
        host, ref = _Host(cfg, 1), safety_ref.Tracker(cfg, 1, 0.1)
        p = [(0, 0, 0), (0.6, 0, 0)]
        _scripted(cfg, host, ref, [(p, [0, 0], p, [(0, 0, 0, 0)] * 2, [prev_clear, 3.0]),
                                   (p, [0, 0], p, [crash, (0, 0, 0, 0)], [3.0, 3.0])])
        assert int(host.state['records'][0, 0, 3]) & 7 == 2 | flag
        assert _bits_equal(host.state['records'], ref.records)


# ------------------------------------------------------------------------------------------------ reduction
def _random_records(rng, R, W, E):
    N = R * W
    count = rng.integers(0, E + 2, N).astype(np.int32)
    results = np.zeros((N, E, 4), np.float32)
    results[:, :, 0] = rng.integers(1, 4, (N, E))
    rec = np.zeros((N, E, 4), np.float32)
    rec[:, :, 0] = rng.uniform(0, 2, (N, E)) * (rng.random((N, E)) < 0.9)
    rec[:, :, 1] = rng.uniform(0, 6, (N, E))
    rec[:, :, 2] = rng.integers(0, 5, (N, E)) * (rng.random((N, E)) < 0.5)
    crashed = results[:, :, 0] == 2
    cause = np.where(crashed, rng.integers(1, 3, (N, E)), 0)
    both = (cause == 2) & (rng.random((N, E)) < 0.5)
    hit = np.where(cause == 2, rng.integers(0, R, (N, E)) + 1, 0)
    rec[:, :, 3] = cause | both * 4 | hit << 8 | rng.integers(0, R + 1, (N, E)) << 16
    return rec, results, count


def test_reduce_equals_the_restatement(built):
    R, W, E = 6, 5, 3
    cfg = _cfg(R=R, W=W)
    rng = np.random.default_rng(5)
    rec, results, count = _random_records(rng, R, W, E)
    mask = (rng.random(R * W) < 0.4).astype(np.uint8)
    got = safety_reduce_host(cfg, rec, results, count)
    want = np.stack([safety_ref.reduce(R, rec, results, count, world=w) for w in range(W)])
    assert _bits_equal(got, want)
    assert got[:, 3].sum() == 0 and got[:, :3].sum() > 0 and got[:, 4].sum() > 0
    split = safety_reduce_host(cfg, rec, results, count, role_mask=mask)
    want2 = np.stack([[safety_ref.reduce(R, rec, results, count, mask, True, want, w) for want in (0, 1)]
                      for w in range(W)])
    assert _bits_equal(split, want2) and split[:, :, 3].sum() > 0
    cols = [i for i in range(13) if i != 3]
    counts = [0, 1, 2, 4, 5, 8, 11, 12]                            # integer columns add up exactly
    assert np.array_equal(split[:, :, counts].sum(1), got[:, counts])
    assert np.allclose(split[:, :, cols].sum(1), got[:, cols], rtol=1e-12)
    assert np.array_equal(split[:, :, 13].min(1), got[:, 13])
    # a sub-range, and totals of two shards: sums in world order, the minimum for the last column
    assert _bits_equal(safety_reduce_host(cfg, rec, results, count, world_begin=2, world_count=2), got[2:4])
    parts = []
    for w0, wc in ((0, 2), (2, 3)):
        c = _cfg(R=R, W=wc)
        sl = slice(w0 * R, (w0 + wc) * R)
        parts.append(safety_reduce_host(c, rec[sl], results[sl], count[sl]))
    tot = safety_totals(got)
    assert _bits_equal(safety_totals(np.concatenate(parts)), tot)
    assert tot[13] == got[:, 13].min() and tot[0] == got[:, 0].sum()


def test_reduce_excludes_infinite_separations(built):
    """R = 1: every record's minimum separation is +inf; it is counted in 'reached' and left out of the sums."""
    cfg = _cfg(R=1, W=3)
    rec = np.zeros((3, 2, 4), np.float32)
    rec[:, :, 0] = np.inf
    rec[:, :, 1] = [[1.0, 2.0], [np.inf, 0.5], [3.0, 3.0]]
    results = np.ones((3, 2, 4), np.float32)
    got = safety_reduce_host(cfg, rec, results, np.int32([2, 2, 1]))
    assert got[:, 4].tolist() == [2, 2, 1] and not got[:, 5:8].any()
    assert got[:, 8].tolist() == [2, 1, 1] and got[:, 9].tolist() == [3.0, 0.5, 3.0]
    assert np.isinf(got[:, 13]).all() and np.isinf(safety_totals(got)[13])


# ------------------------------------------------------------------------------------------------ rejections
def test_abi_rejects_bad_arguments(built):
    lib = _lib.load()
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    R, W, E = 3, 2, 2
    cfg = _cfg(R=R, W=W, beams=8)
    N = R * W
    f = lambda *s: np.zeros(s, np.float32)
    i = lambda *s: np.zeros(s, np.int32)
    bufs = [f(N, 4), i(N, 4), f(N, 4), np.zeros((N, 4), np.uint8), f(N, 8), i(N), i(N)]
    state = [f(N), f(N), f(N), i(N), i(N), f(N, E, 4)]
    good = _lib.SafetyParams(0.1)
    track = lambda c, p, b, e, s: lib.rlca_safety_track_host(c, p, *[None if x is None else vp(x) for x in b], e,
                                                             *[None if x is None else vp(x) for x in s])
    assert track(C.byref(cfg), C.byref(good), bufs, E, state) == 0
    for k in range(len(bufs)):
        bad = list(bufs)
        bad[k] = None
        assert track(C.byref(cfg), C.byref(good), bad, E, state) == 1, k
    for k in range(len(state)):
        bad = list(state)
        bad[k] = None
        assert track(C.byref(cfg), C.byref(good), bufs, E, bad) == 1, k
    assert track(None, C.byref(good), bufs, E, state) == 1
    assert track(C.byref(cfg), None, bufs, E, state) == 1
    assert track(C.byref(cfg), C.byref(good), bufs, 0, state) == 1
    bad_near = (math.nan, -1.0, math.inf, -math.inf)
    for d in bad_near:
        assert track(C.byref(cfg), C.byref(_lib.SafetyParams(d)), bufs, E, state) == 1, d
        assert b'near_dist' in lib.rlca_last_error()
    assert track(C.byref(cfg), C.byref(_lib.SafetyParams(0.0)), bufs, E, state) == 0
    for K in (0, 65, -1):
        c = _cfg(R=K, W=W, beams=8)
        assert track(C.byref(c), C.byref(good), bufs, E, state) == 1, K
    # the host reduction
    rec, res, cnt, out = f(N, E, 4), f(N, E, 4), i(N), np.zeros((W, 14))
    red = lambda c, a, b, n, e, w0, wc, o: lib.rlca_safety_reduce_host(c, a, b, n, None, e, w0, wc, o)
    assert red(C.byref(cfg), vp(rec), vp(res), vp(cnt), E, 0, W, vp(out)) == 0
    assert red(None, vp(rec), vp(res), vp(cnt), E, 0, W, vp(out)) == 1
    assert red(C.byref(cfg), None, vp(res), vp(cnt), E, 0, W, vp(out)) == 1
    assert red(C.byref(cfg), vp(rec), None, vp(cnt), E, 0, W, vp(out)) == 1
    assert red(C.byref(cfg), vp(rec), vp(res), None, E, 0, W, vp(out)) == 1
    assert red(C.byref(cfg), vp(rec), vp(res), vp(cnt), E, 0, W, None) == 1
    assert red(C.byref(cfg), vp(rec), vp(res), vp(cnt), 0, 0, W, vp(out)) == 1
    for w0, wc in ((-1, 1), (0, 0), (1, W), (W, 1)):
        assert red(C.byref(cfg), vp(rec), vp(res), vp(cnt), E, w0, wc, vp(out)) == 1, (w0, wc)
    # the device entries check their arguments before they launch anything
    st = _lib.EnvState(vp(bufs[0]), vp(bufs[0]), vp(bufs[0]), vp(bufs[1]))
    io = _lib.StepIO(None, None, vp(bufs[4]), None, vp(bufs[3]), None, None, None, None)
    ev = _lib.EvalState(None, vp(bufs[6]), vp(bufs[5]), vp(bufs[5]), vp(res), E)
    ss = _lib.SafetyState(*[vp(x) for x in state], E)
    dev = lambda c, p, s0, s1, o, e, s: lib.rlca_safety_track(c, p, s0, s1, o, e, s, None)
    ok = [C.byref(cfg), C.byref(good), C.byref(st), C.byref(st), C.byref(io), C.byref(ev), C.byref(ss)]
    for k in range(len(ok)):
        bad = list(ok)
        bad[k] = None
        assert dev(*bad) == 1, k
    for d in bad_near:
        assert dev(ok[0], C.byref(_lib.SafetyParams(d)), *ok[2:]) == 1, d
    assert dev(*ok[:5], C.byref(_lib.EvalState(None, vp(bufs[6]), vp(bufs[5]), vp(bufs[5]), vp(res), E + 1)), ok[6]) == 1
    assert b'different number of episodes' in lib.rlca_last_error()
    for field in ('min_sep_dev', 'min_clear_dev', 'last_clear_dev', 'near_dev', 'partner_dev', 'records_dev'):
        s2 = _lib.SafetyState(*[vp(x) for x in state], E)
        setattr(s2, field, None)
        assert dev(*ok[:6], C.byref(s2)) == 1, field
    io2 = _lib.StepIO(None, None, None, None, vp(bufs[3]), None, None, None, None)
    assert dev(*ok[:4], C.byref(io2), *ok[5:]) == 1
    dred = lambda c, s, e, o, w0=0, wc=W: lib.rlca_safety_reduce(c, s, e, None, w0, wc, o, None)
    assert dred(None, C.byref(ss), C.byref(ev), vp(out)) == 1
    assert dred(C.byref(cfg), None, C.byref(ev), vp(out)) == 1
    assert dred(C.byref(cfg), C.byref(ss), None, vp(out)) == 1
    assert dred(C.byref(cfg), C.byref(ss), C.byref(ev), None) == 1
    assert dred(C.byref(cfg), C.byref(ss), C.byref(ev), vp(out), 1, W) == 1
    sep = lambda c, a, b, n, o: lib.rlca_safety_separation_host(c, a, b, n, o)
    assert sep(C.byref(cfg), vp(bufs[0]), vp(bufs[0]), N, vp(state[0])) == 0
    assert sep(C.byref(cfg), None, vp(bufs[0]), N, vp(state[0])) == 1
    assert sep(C.byref(cfg), vp(bufs[0]), vp(bufs[0]), -1, vp(state[0])) == 1
    assert lib.rlca_safety_contact_host(C.byref(cfg), None) == 1


def test_python_wrappers_reject(built):
    from rl_collision_avoidance_b200.evaluation import SafetyTracker
    for d in (math.nan, -0.5, math.inf):
        with pytest.raises(ValueError, match='near_dist'):
            SafetyTracker(None, None, d)


@pytest.mark.parametrize('value', ['nan', '-1', 'inf'])
def test_evaluate_cli_rejects_bad_near_miss(capsys, value):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(['--scenario', 'stage2', '--policy', os.path.join(CKPT, 'stage2.pth'), '--near-miss', value])
    assert e.value.code == 2
    assert '--near-miss must be finite and >= 0' in capsys.readouterr().err


def test_kernel_does_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_safety.o')], check=True,
                         capture_output=True, text=True).stdout
    for name, regs in (('rlca_safety_track_kernel', 64), ('rlca_safety_reduce_kernel', 64)):
        m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)' % name, out)
        assert m, out
        assert int(m.group(2)) == 0 and int(m.group(4)) == 0, m.group(0)
        assert int(m.group(1)) <= regs, m.group(0)
