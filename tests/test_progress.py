"""Progress metrics without a GPU (DESIGN.md §9o): the host twin of csrc/rlca_progress.cu against the numpy
restatement (tests/progress_ref.py) on scripted sequences and oracle rollouts; the cause of each scripted time-out;
the reduction, split and sharded; every rejected argument; the kernels' registers."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import progress_ref
from helpers import make_pair, random_actions
from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.evaluation import PROGRESS_COLUMNS, progress_metrics, progress_reduce_host, \
    progress_totals, progress_track_host
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
_F = np.float32
NONE, TIMEOUT, TIMEOUT_RESPAWN, REACH = (0, 0, 0, 0), (1, 0, 3, 0), (1, 0, 3, 1), (1, 0, 1, 0)


def _cfg(R=1, W=1, scenario='circle', auto_reset=0):
    sc = make_scenario(scenario)
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=W, beams=8, auto_reset=auto_reset)
    cfg.robots_per_world = R
    return cfg


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


class _Host:
    """rlca_progress_track_host next to a host copy of the episode tracker's boundaries, and the restatement."""

    def __init__(self, cfg, episodes, **params):
        self.cfg, self.E, self.params = cfg, episodes, params
        N = cfg.robots_per_world * cfg.num_worlds
        self.closed = np.full(N, -1, np.int32)
        self.count = np.zeros(N, np.int32)
        self.open = np.ones(N, np.int32)
        self.results = np.zeros((N, episodes, 4), np.float32)
        self.state = dict(running=np.zeros((N, 4), np.float32), counters=np.zeros((N, 4), np.int32),
                          records=np.zeros((N, episodes, 4), np.float32), causes=np.zeros((N, episodes), np.uint8))
        self.ref = progress_ref.Tracker(cfg, episodes, **params)

    def tick(self, pose_in, meta_in, pose_out, flags, meta_out):
        progress_track_host(self.cfg, self.params, pose_in, meta_in, pose_out, flags, self.closed, self.count,
                            self.state)
        self.ref.tick(pose_in, meta_in, pose_out, flags, meta_out)
        for a in np.nonzero((self.closed != meta_in[:, 1]) & (flags[:, 2] != 0))[0]:      # the episode tracker's rule
            if self.count[a] < self.E:
                self.results[a, self.count[a], 0] = flags[a, 2]
            self.count[a] += 1
            self.closed[a] = meta_in[a, 1]
        self.open[:] = self.closed != meta_out[:, 1]

    def check(self):
        for k, v in self.ref.state().items():
            assert _bits_equal(self.state[k], v), k
        assert np.array_equal(self.count, self.ref.count) and np.array_equal(self.closed, self.ref.closed)
        assert np.array_equal(self.open, self.ref.open)

    def partials(self, **kw):
        return progress_reduce_host(self.cfg, self.params, self.state, self.results, self.count, self.open, **kw)

    def ref_partials(self, w=0):
        st = self.ref.state()
        return progress_ref.reduce(self.ref.window, self.cfg.robots_per_world, st['records'], st['causes'],
                                   st['running'], st['counters'], self.ref.results, self.ref.count, self.ref.open,
                                   world=w)


def _script(host, steps):
    """steps: (pose_in, ep_in, pose_out, flags, ep_out) per tick, poses (R, 4) x, y, theta, distance to the goal."""
    for pose_in, ep_in, pose_out, flags, ep_out in steps:
        R = len(pose_in)
        mi, mo = np.zeros((R, 4), np.int32), np.zeros((R, 4), np.int32)
        mi[:, 1], mo[:, 1] = ep_in, ep_out
        host.tick(_F(pose_in), mi, _F(pose_out), np.asarray(flags, np.uint8), mo)
    host.check()


def _path(poses, last_flags=TIMEOUT, ep=0, next_ep=None, respawn_pose=None):
    """One robot's ticks along `poses` ((x, y, theta, d) per pose), the last tick ending the episode with `last_flags`
    (and on a re-spawn moving it to `respawn_pose`, episode next_ep)."""
    steps = []
    for t in range(len(poses) - 1):
        last = t == len(poses) - 2
        out = poses[t + 1]
        fl, ep_out = NONE, ep
        if last:
            fl = last_flags
            if fl[3]:
                out, ep_out = respawn_pose, next_ep
        steps.append(([poses[t]], [ep], [out], [fl], [ep_out]))
    return steps


def _record(host, a=0, i=0):
    rec = host.state['records'][a, i]
    return float(rec[0]), float(rec[1]), int(rec[2]), int(rec[3]), int(host.state['causes'][a, i])


# ------------------------------------------------------------------------------------------------ header
def test_column_names_follow_the_header(built):
    src = open(os.path.join(ROOT, 'include', 'rlca.h')).read()
    idx = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r'#define RLCA_PROGRESS_([A-Z_]+) (\d+)', src)}
    assert idx.pop('npartials') == len(PROGRESS_COLUMNS) == len(progress_ref.COLUMNS)
    assert sorted(idx.values()) == list(range(len(PROGRESS_COLUMNS)))
    for name, i in idx.items():
        assert PROGRESS_COLUMNS[i] == name, (name, i)
    assert PROGRESS_COLUMNS == progress_ref.COLUMNS


# ------------------------------------------------------------------------------------------------ scripted fold
def test_frozen_from_the_first_tick(built):
    host = _Host(_cfg(), 1, window=5)
    _script(host, _path([(1.0, 2.0, 0.5, 4.0)] * 9))
    assert _record(host) == (4.0, 0.0, 8, 8, 1)
    assert not host.state['running'].any() and not host.state['counters'].any()      # reset after the end


def test_turning_in_place_is_frozen_with_rotation(built):
    host = _Host(_cfg(), 1, window=5)
    poses, th = [], _F(2.5)
    for t in range(12):                                            # 0.3 rad per tick, across the +-pi seam
        poses.append((1.0, 2.0, float(th), 4.0))
        th = progress_ref.wrap(_F(th + _F(0.3)))
    _script(host, _path(poses))
    closest, rot, still, ticks, cause = _record(host)
    assert cause == 1 and still == ticks == 11
    assert abs(rot - 11 * 0.3) < 1e-4, rot


def test_circling_is_stalled(built):
    """1 m radius round the goal at 0.1 m per tick: moving, never closer."""
    host = _Host(_cfg(), 1, window=20)
    poses = []
    for t in range(60):
        a = 0.1 * t
        poses.append((3.0 + math.cos(a), 4.0 + math.sin(a), a + math.pi / 2, 1.0))
    _script(host, _path(poses))
    closest, rot, still, ticks, cause = _record(host)
    assert cause == 2 and still == 0 and ticks == 59 and closest == 1.0
    assert abs(rot - 5.9) < 1e-3


def test_driving_too_slowly_is_slow(built):
    """0.02 m per tick straight at the goal: 0.1 m of progress every 5 ticks, inside a window of 10."""
    host = _Host(_cfg(), 1, window=10)
    poses = [(0.02 * t, 0.0, 0.0, 10.0 - 0.02 * t) for t in range(80)]
    _script(host, _path(poses))
    closest, rot, still, ticks, cause = _record(host)
    assert cause == 3 and still == 0 and rot == 0.0 and abs(closest - (10.0 - 0.02 * 79)) < 1e-4


def test_exact_boundaries(built):
    """d lands exactly on ref - progress_dist (progress: <=) and s exactly on still_dist (moving: <), every tick; a
    window of one tick makes a single miss decide the cause."""
    host = _Host(_cfg(), 1, window=1, progress_dist=0.25, still_dist=0.25)
    poses = [(0.25 * t, 0.0, 0.0, 2.0 - 0.25 * t) for t in range(5)]
    _script(host, _path(poses))
    assert _record(host) == (1.0, 0.0, 0, 4, 3)
    # one ulp short of the progress boundary, moving 0.25 m a tick: stalled
    host = _Host(_cfg(), 1, window=1, progress_dist=0.25, still_dist=0.25)
    short = float(np.nextafter(_F(1.75), _F(2)))
    poses = [(0.25 * t, 0.0, 0.0, 2.0 if t < 2 else short) for t in range(6)]
    _script(host, _path(poses))
    assert _record(host)[2:] == (0, 5, 2)
    # one ulp short of the still boundary, progressing exactly 0.25 m a tick: frozen
    host = _Host(_cfg(), 1, window=1, progress_dist=0.25, still_dist=0.25)
    step = float(np.nextafter(_F(0.25), _F(0)))
    poses = [(step * (t & 1), 0.0, 0.0, 2.0 - 0.25 * t) for t in range(6)]
    _script(host, _path(poses))
    assert _record(host)[2:] == (5, 5, 1)


def test_time_out_on_a_re_spawn_tick_uses_the_previous_state(built):
    """Stage 1: the time-out tick re-spawns the robot; state_out holds the next episode, which must not count."""
    host = _Host(_cfg(auto_reset=1), 2, window=4)
    poses = [(1.0, 1.0, 0.0, 3.0)] * 6
    _script(host, _path(poses, TIMEOUT_RESPAWN, 0, 1, (9.0, 9.0, 1.0, 0.5)))
    assert _record(host) == (3.0, 0.0, 4, 4, 1)
    assert host.count[0] == 1 and host.open[0] == 1
    assert not host.state['counters'].any()                        # the new episode has no folded tick yet
    # its first tick is its own
    _script(host, [([(9.0, 9.0, 1.0, 0.5)], [1], [(9.0, 9.0, 1.0, 0.5)], [NONE], [1])])
    assert host.state['counters'][0].tolist() == [0, 1, 1, 1] and host.state['running'][0, 0] == _F(0.5)


def test_idle_ticks_and_repeated_terminations_add_nothing(built):
    """Stage 2 / circle: after its end a robot idles (or stays terminal) in the same episode; nothing is folded or
    recorded until its group re-spawns it."""
    host = _Host(_cfg(auto_reset=2), 3, window=4)
    p, q = (1.0, 1.0, 0.0, 3.0), (1.5, 1.0, 0.0, 2.5)
    steps = _path([p, q, q], REACH)
    steps += [([q], [0], [q], [(1, 0, 1, 0)], [0])] * 3             # repeated terminations (circle)
    steps += [([q], [0], [(q[0] + 0.5, 1.0, 2.0, 2.0)], [NONE], [0])] * 3   # idling on its last command (stage 2)
    steps += [([q], [0], [(5.0, 5.0, 0.0, 7.0)], [(0, 0, 0, 1)], [1])]       # the group re-spawns
    steps += _path([(5.0, 5.0, 0.0, 7.0)] * 6, TIMEOUT, 1)
    _script(host, steps)
    assert host.count[0] == 2 and host.results[0, :2, 0].tolist() == [1, 3]
    assert _record(host, 0, 0) == (2.5, 0.0, 1, 2, 0)             # the second tick stood still
    assert _record(host, 0, 1) == (7.0, 0.0, 5, 5, 1)


def test_episodes_after_the_last_slot_are_counted_and_dropped(built):
    host = _Host(_cfg(auto_reset=1), 2, window=2)
    steps = []
    for ep in range(4):
        d = 5.0 + ep
        steps += _path([(0.0, 0.0, 0.0, d)] * 4, TIMEOUT_RESPAWN, ep, ep + 1, (0.0, 0.0, 0.0, d + 1))
    _script(host, steps)
    assert host.count[0] == 4
    assert [_record(host, 0, i) for i in range(2)] == [(5.0, 0.0, 2, 2, 1), (6.0, 0.0, 2, 2, 1)]


def test_robot_near_counts_parked_robots_and_never_fires_alone(built):
    """Robot 1 reached its goal and stands parked 0.5 m from robot 0, which times out frozen: frozen + 4.  With a
    block distance below 0.5 m, or alone in its world (R = 1), it is frozen only."""
    stay0, stay1 = (0.0, 0.0, 0.0, 3.0), (0.5, 0.0, 0.0, 0.1)
    for block, want in ((1.0, 5), (0.5, 1)):
        host = _Host(_cfg(R=2), 1, window=3, block_dist=block)
        steps = [([stay0, stay1], [0, 0], [stay0, stay1], [NONE, REACH], [0, 0])]
        steps += [([stay0, stay1], [0, 0], [stay0, stay1], [NONE, (1, 0, 1, 0)], [0, 0])] * 3
        steps += [([stay0, stay1], [0, 0], [stay0, stay1], [TIMEOUT, (1, 0, 1, 0)], [0, 0])]
        _script(host, steps)
        assert host.count.tolist() == [1, 1] and host.closed.tolist() == [0, 0]
        assert _record(host, 0)[4] == want, block
        assert _record(host, 1)[4] == 0
    host = _Host(_cfg(R=1, W=2), 1, window=3)
    steps = [([stay0, stay1], [0, 0], [stay0, stay1], [NONE, NONE], [0, 0])] * 3
    steps += [([stay0, stay1], [0, 0], [stay0, stay1], [TIMEOUT, TIMEOUT], [0, 0])]
    _script(host, steps)
    assert host.state['causes'][:, 0].tolist() == [1, 1]


def test_unfinished_episodes_are_classified_at_the_reduction(built):
    """Still running when evaluation stops: robot 0 frozen with robot 1 near, robot 1 driving at the goal 0.125 m per
    tick next to it, and robot 2, which circled until its time-out re-spawned it on the last tick (stalled), so that
    its new episode has no folded tick (slow, left out of the closest sums)."""
    host = _Host(_cfg(R=3, auto_reset=1), 2, window=3)
    a = (0.0, 0.0, 0.0, 3.0)
    for t in range(5):
        b0 = (0.25 + 0.125 * t, 0.0, 0.0, 4.0 - 0.125 * t)
        b1 = (0.25 + 0.125 * (t + 1), 0.0, 0.0, 4.0 - 0.125 * (t + 1))
        c0 = (10.0 + math.cos(0.2 * t), math.sin(0.2 * t), 0.0, 1.0)
        c1 = (10.0 + math.cos(0.2 * t + 0.2), math.sin(0.2 * t + 0.2), 0.0, 1.0)
        last = t == 4
        _script(host, [([a, b0, c0], [0, 0, 0], [a, b1, (20.0, 20.0, 0.0, 8.0) if last else c1],
                        [NONE, NONE, TIMEOUT_RESPAWN if last else NONE], [0, 0, 1 if last else 0])])
    got = host.partials()[0]
    assert _bits_equal(got, host.ref_partials())
    t = dict(zip(PROGRESS_COLUMNS, got.tolist()))
    assert (t['timeout_frozen'], t['timeout_stalled'], t['timeout_slow'], t['timeout_robot_near']) == (0, 1, 0, 0)
    assert (t['timeout_folded'], t['timeout_sum_closest']) == (1, 1.0)
    assert (t['unfinished_frozen'], t['unfinished_stalled'], t['unfinished_slow']) == (1, 0, 2)
    assert (t['unfinished_robot_near'], t['unfinished_folded'], t['unfinished_sum_closest']) == (2, 2, 3.0 + 3.375)
    assert (t['sum_still_ticks'], t['sum_ticks'], t['reached']) == (0, 4, 0)
    m = progress_metrics(progress_totals(got))
    assert m['timeouts'] == 1 and m['unfinished'] == 3 and m['timeout_stalled_share'] == 1.0
    assert m['unfinished_closest'][0] == (3.0 + 3.375) / 2 and m['still_share'] == 0.0


# ------------------------------------------------------------------------------------------------ oracle rollouts
def _env_cfg(orc):
    cfg = _lib.EnvConfig()
    for name, _ in cfg._fields_:
        setattr(cfg, name, getattr(orc.cfg, name))
    return cfg


@pytest.mark.parametrize('scenario,auto_reset,R', [('stage1', 1, None), ('stage2', 2, None), ('circle', 0, 6)])
def test_host_twin_equals_the_restatement_on_oracle_rollouts(built, scenario, auto_reset, R):
    """Random actions on the oracle with a short time-out budget: every tick's running state and records bit-equal."""
    sc, _, orc = make_pair(scenario, num_worlds=2, beams=32, auto_reset=auto_reset, gpu=False, robots_per_world=R,
                           radius=3.0 if scenario == 'circle' else None, seed=11)
    orc.reset_world()
    orc.reset_pose()
    cfg = _env_cfg(orc)
    host = _Host(cfg, 3, window=8, progress_dist=0.1, still_dist=0.01, block_dist=1.5)
    rng = np.random.default_rng(12)
    for t in range(160):
        pose_in, meta_in = orc.pose.copy(), orc.meta.copy()
        act = random_actions(rng, orc.N)
        act[::3, 0] = 0.0                                          # some robots stand still
        orc.step(act)
        host.tick(pose_in, meta_in, orc.pose, orc.flags, orc.meta)
        if t % 40 == 39:
            host.check()
    assert host.count.sum() > 0
    assert np.array_equal((host.state['causes'] != 0), host.results[:, :, 0] == 3)
    W = cfg.num_worlds
    got = host.partials()
    assert _bits_equal(got, np.stack([host.ref_partials(w) for w in range(W)]))


# ------------------------------------------------------------------------------------------------ reduction
def _random_state(rng, R, W, E):
    N = R * W
    count = rng.integers(0, E + 2, N).astype(np.int32)
    open_ = rng.integers(0, 2, N).astype(np.int32)
    results = np.zeros((N, E, 4), np.float32)
    results[:, :, 0] = rng.integers(1, 4, (N, E))
    rec = np.zeros((N, E, 4), np.float32)
    rec[:, :, 0] = rng.uniform(0, 8, (N, E))
    rec[:, :, 1] = rng.uniform(0, 30, (N, E))
    rec[:, :, 3] = rng.integers(0, 300, (N, E))
    rec[:, :, 2] = np.floor(rec[:, :, 3] * rng.random((N, E)))
    causes = np.where(results[:, :, 0] == 3, rng.integers(1, 4, (N, E)) + 4 * rng.integers(0, 2, (N, E)), 0)
    running = np.zeros((N, 4), np.float32)
    running[:, 0] = rng.uniform(0, 8, N)
    running[:, 3] = rng.integers(0, 2, N)
    counters = rng.integers(0, 12, (N, 4)).astype(np.int32)
    counters[rng.random(N) < 0.2] = 0
    state = dict(records=rec, causes=causes.astype(np.uint8), running=running, counters=counters)
    return state, results, count, open_


def test_reduce_equals_the_restatement(built):
    R, W, E, window = 6, 5, 3, 6
    cfg = _cfg(R=R, W=W)
    params = {'window': window}
    rng = np.random.default_rng(5)
    st, results, count, open_ = _random_state(rng, R, W, E)
    mask = (rng.random(R * W) < 0.4).astype(np.uint8)
    ref = lambda w, **kw: progress_ref.reduce(window, R, st['records'], st['causes'], st['running'], st['counters'],
                                              results, count, open_, world=w, **kw)
    got = progress_reduce_host(cfg, params, st, results, count, open_)
    assert _bits_equal(got, np.stack([ref(w) for w in range(W)]))
    assert (got[:, :4] > 0).any() and (got[:, 7:11] > 0).any() and (got[:, 16] > 0).any()
    # the causes add up to the tracker's time-outs and unfinished episodes
    n = np.minimum(count, E)
    timeouts = [sum(int((results[a, :n[a], 0] == 3).sum()) for a in range(w * R, (w + 1) * R)) for w in range(W)]
    unfinished = [int(((count < E) & (open_ != 0))[w * R:(w + 1) * R].sum()) for w in range(W)]
    assert got[:, 0:3].sum(1).tolist() == timeouts and got[:, 7:10].sum(1).tolist() == unfinished
    split = progress_reduce_host(cfg, params, st, results, count, open_, role_mask=mask)
    want2 = np.stack([[ref(w, mask=mask, split=True, want=v) for v in (0, 1)] for w in range(W)])
    assert _bits_equal(split, want2)
    counts = [0, 1, 2, 3, 4, 7, 8, 9, 10, 11, 14, 15, 16]           # integer columns add up exactly
    assert np.array_equal(split[:, :, counts].sum(1), got[:, counts])
    assert np.allclose(split.sum(1), got, rtol=1e-12)
    # a sub-range, and totals of two shards in world order
    assert _bits_equal(progress_reduce_host(cfg, params, st, results, count, open_, world_begin=2, world_count=2),
                       got[2:4])
    parts = []
    for w0, wc in ((0, 2), (2, 3)):
        sl = slice(w0 * R, (w0 + wc) * R)
        parts.append(progress_reduce_host(_cfg(R=R, W=wc), params, {k: v[sl] for k, v in st.items()}, results[sl],
                                          count[sl], open_[sl]))
    assert _bits_equal(progress_totals(np.concatenate(parts)), progress_totals(got))
    # a longer window moves frozen / stalled unfinished episodes to slow, and leaves the records' causes alone
    longer = progress_reduce_host(cfg, {'window': 100}, st, results, count, open_)
    assert _bits_equal(longer[:, :7], got[:, :7]) and longer[:, 7:9].sum() == 0


def test_metrics(built):
    tot = np.zeros(len(PROGRESS_COLUMNS))
    t = dict(zip(PROGRESS_COLUMNS, range(len(PROGRESS_COLUMNS))))
    tot[[t['timeout_frozen'], t['timeout_stalled'], t['timeout_slow'], t['timeout_robot_near']]] = [1, 2, 1, 2]
    tot[[t['timeout_folded'], t['timeout_sum_closest'], t['timeout_sum_closest_sq']]] = [4, 8.0, 20.0]
    tot[[t['sum_still_ticks'], t['sum_ticks'], t['reached'], t['sum_rotation'], t['sum_rotation_sq']]] = \
        [25, 100, 2, 6.0, 20.0]
    m = progress_metrics(tot)
    assert m['timeouts'] == 4 and m['timeout_stalled_share'] == 0.5 and m['timeout_robot_near_share'] == 0.5
    assert m['timeout_closest'] == (2.0, 1.0) and m['still_share'] == 0.25 and m['rotation_reached'] == (3.0, 1.0)
    assert m['unfinished'] == 0 and math.isnan(m['unfinished_frozen_share'])
    assert all(math.isnan(v) for v in m['unfinished_closest'])


# ------------------------------------------------------------------------------------------------ rejections
def test_abi_rejects_bad_arguments(built):
    lib = _lib.load()
    vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
    R, W, E = 3, 2, 2
    cfg = _cfg(R=R, W=W)
    N = R * W
    f = lambda *s: np.zeros(s, np.float32)
    i = lambda *s: np.zeros(s, np.int32)
    bufs = [f(N, 4), i(N, 4), f(N, 4), np.zeros((N, 4), np.uint8), i(N), i(N)]
    state = [f(N, 4), i(N, 4), f(N, E, 4), np.zeros((N, E), np.uint8)]
    good = _lib.ProgressParams(50, 0.1, 0.005, 1.0)
    track = lambda c, p, b, e, s: lib.rlca_progress_track_host(c, p, *[vp(x) for x in b], e, *[vp(x) for x in s])
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
    bad_params = [_lib.ProgressParams(0, 0.1, 0.005, 1.0), _lib.ProgressParams(-3, 0.1, 0.005, 1.0)]
    for field in ('progress_dist', 'still_dist', 'block_dist'):
        for v in (math.nan, -1.0, math.inf, -math.inf):
            p = _lib.ProgressParams(50, 0.1, 0.005, 1.0)
            setattr(p, field, v)
            bad_params.append(p)
    for p in bad_params:
        assert track(C.byref(cfg), C.byref(p), bufs, E, state) == 1, (p.window, p.progress_dist, p.still_dist,
                                                                       p.block_dist)
    assert track(C.byref(cfg), C.byref(_lib.ProgressParams(1, 0.0, 0.0, 0.0)), bufs, E, state) == 0
    for K in (0, 65, -1):
        assert track(C.byref(_cfg(R=K, W=W)), C.byref(good), bufs, E, state) == 1, K
    # the host reduction
    rec, res, cnt, opn, out = f(N, E, 4), f(N, E, 4), i(N), i(N), np.zeros((W, len(PROGRESS_COLUMNS)))
    red_args = [vp(state[2]), vp(state[3]), vp(state[0]), vp(state[1]), vp(res), vp(cnt), vp(opn)]
    red = lambda c, p, a, e=E, w0=0, wc=W, o=vp(out): lib.rlca_progress_reduce_host(c, p, *a, None, e, w0, wc, o)
    assert red(C.byref(cfg), C.byref(good), red_args) == 0
    assert red(None, C.byref(good), red_args) == 1
    assert red(C.byref(cfg), None, red_args) == 1
    for k in range(len(red_args)):
        bad = list(red_args)
        bad[k] = None
        assert red(C.byref(cfg), C.byref(good), bad) == 1, k
    assert red(C.byref(cfg), C.byref(good), red_args, o=None) == 1
    assert red(C.byref(cfg), C.byref(good), red_args, e=0) == 1
    for p in bad_params:
        assert red(C.byref(cfg), C.byref(p), red_args) == 1
    for w0, wc in ((-1, 1), (0, 0), (1, W), (W, 1)):
        assert red(C.byref(cfg), C.byref(good), red_args, w0=w0, wc=wc) == 1, (w0, wc)
    # the device entries check their arguments before they launch anything
    st = _lib.EnvState(vp(bufs[0]), vp(bufs[0]), vp(bufs[0]), vp(bufs[1]))
    io = _lib.StepIO(None, None, None, None, vp(bufs[3]), None, None, None, None)
    ev = _lib.EvalState(None, vp(bufs[5]), vp(bufs[4]), vp(bufs[4]), vp(res), E)
    ps = _lib.ProgressState(*[vp(x) for x in state], E)
    dev = lambda c, p, s0, s1, o, e, s: lib.rlca_progress_track(c, p, s0, s1, o, e, s, None)
    ok = [C.byref(cfg), C.byref(good), C.byref(st), C.byref(st), C.byref(io), C.byref(ev), C.byref(ps)]
    for k in range(len(ok)):
        bad = list(ok)
        bad[k] = None
        assert dev(*bad) == 1, k
    for p in bad_params:
        assert dev(ok[0], C.byref(p), *ok[2:]) == 1
    ev2 = _lib.EvalState(None, vp(bufs[5]), vp(bufs[4]), vp(bufs[4]), vp(res), E + 1)
    assert dev(*ok[:5], C.byref(ev2), ok[6]) == 1
    assert b'different number of episodes' in lib.rlca_last_error()
    for field in ('running_dev', 'counters_dev', 'records_dev', 'causes_dev'):
        s2 = _lib.ProgressState(*[vp(x) for x in state], E)
        setattr(s2, field, None)
        assert dev(*ok[:6], C.byref(s2)) == 1, field
    io2 = _lib.StepIO(None, None, None, None, None, None, None, None, None)
    assert dev(*ok[:4], C.byref(io2), *ok[5:]) == 1
    for field in ('closed_dev', 'count_dev'):
        e2 = _lib.EvalState(None, vp(bufs[5]), vp(bufs[4]), vp(bufs[4]), vp(res), E)
        setattr(e2, field, None)
        assert dev(*ok[:5], C.byref(e2), ok[6]) == 1, field
    dred = lambda c, p, s, e, o, w0=0, wc=W: lib.rlca_progress_reduce(c, p, s, e, None, w0, wc, o, None)
    args = [C.byref(cfg), C.byref(good), C.byref(ps), C.byref(ev), vp(out)]
    for k in range(len(args)):
        bad = list(args)
        bad[k] = None
        assert dred(*bad) == 1, k
    assert dred(*args, w0=1, wc=W) == 1
    assert dred(*args[:3], C.byref(ev2), args[4]) == 1
    e3 = _lib.EvalState(None, vp(bufs[5]), vp(bufs[4]), None, vp(res), E)
    assert dred(*args[:3], C.byref(e3), args[4]) == 1


def test_python_wrappers_reject(built):
    from rl_collision_avoidance_b200.evaluation import ProgressTracker, progress_params
    for bad in ({'window': 0}, {'window': 2.5}, {'progress_dist': math.nan}, {'still_dist': -0.1},
                {'block_dist': math.inf}, {'windw': 3}):
        with pytest.raises(ValueError):
            ProgressTracker(None, None, bad)
    p = progress_params({'window': 7})
    assert (p.window, p.block_dist) == (7, 1.0)


@pytest.mark.parametrize('value', ['0', '-2'])
def test_evaluate_cli_rejects_bad_stall_window(capsys, value):
    import evaluate
    with pytest.raises(SystemExit) as e:
        evaluate.main(['--scenario', 'stage2', '--policy', os.path.join(CKPT, 'stage2.pth'), '--stall-window', value])
    assert e.value.code == 2
    assert '--stall-window must be >= 1' in capsys.readouterr().err


def test_kernels_do_not_spill(built):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', 'rlca_progress.o')], check=True,
                         capture_output=True, text=True).stdout
    for name, regs in (('rlca_progress_track_kernel', 64), ('rlca_progress_reduce_kernel', 96)):
        m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)' % name, out)
        assert m, out
        assert int(m.group(2)) == 0 and int(m.group(4)) == 0, m.group(0)
        assert int(m.group(1)) <= regs, m.group(0)
