"""Evaluation on the device (csrc/rlca_eval.cu, rl_collision_avoidance_b200/evaluation.py): episode records against
the CPU oracle's ticks, the stage-2 idle ticks, evaluate() with the shipped checkpoints, determinism and shard
invariance of the float64 partials, and circle layouts with K != 50 robots against the oracle."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, random_actions
from oracle.oracle import OracleWorld, OrcConfig
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _pair(sc, worlds, auto_reset, seed, world_offset=0):
    from rl_collision_avoidance_b200.stage_world import StageWorld
    ocfg = fill_config(OrcConfig(), sc, num_worlds=worlds, beams=512, auto_reset=auto_reset, seed=seed,
                       world_offset=world_offset)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    env = StageWorld(512, index=0, scenario=sc, num_worlds=worlds, seed=seed, auto_reset=auto_reset,
                     world_offset=world_offset)
    return env, orc


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cpu'))
    return pol


class _HostRecords:
    """The records the tracker must produce, from the oracle's ticks: the first termination of each episode index,
    path = float64 polyline through the oracle's poses; on a tick that re-spawned the robot the last segment is
    |v_clip| dt, or 0 when it crashed."""

    def __init__(self, n, dt, vmin, vmax):
        self.path = np.zeros(n)
        self.closed = np.full(n, -1)
        self.rec = [[] for _ in range(n)]
        self.dt, self.vmin, self.vmax = float(np.float32(dt)), vmin, vmax

    def tick(self, pose0, ep0, action, pose1, flags, eplog):
        for a in range(len(self.path)):
            fl = flags[a]
            if self.closed[a] != ep0[a]:
                if fl[3]:
                    v = float(np.clip(action[a, 0], self.vmin, self.vmax))
                    seg = 0.0 if fl[1] else abs(v) * self.dt
                else:
                    seg = float(np.hypot(np.float64(pose1[a, 0]) - pose0[a, 0], np.float64(pose1[a, 1]) - pose0[a, 1]))
                self.path[a] += seg
                if fl[2]:
                    e = eplog[a].astype(np.float64)
                    straight = np.float32(np.sqrt((e[0] - e[4]) ** 2 + (e[1] - e[5]) ** 2))
                    self.rec[a].append((int(e[6]), int(e[3]), self.path[a], straight))
                    self.closed[a] = ep0[a]
                    self.path[a] = 0.0
            if fl[3]:
                self.path[a] = 0.0


def _check_records(tracker, ref, E):
    torch.cuda.synchronize()
    count = tracker.count.cpu().numpy()
    recs = tracker.records.cpu().numpy()
    n_rec = 0
    for a, rows in enumerate(ref.rec):
        assert count[a] == len(rows), (a, count[a], len(rows))
        for i, (res, ticks, path, straight) in enumerate(rows[:E]):
            got = recs[a, i]
            assert got[0] == res and got[1] == ticks, (a, i, got, res, ticks)
            assert got[3] == straight, (a, i, got[3], straight)
            assert abs(float(got[2]) - path) <= 1e-5 * path + 1e-6, (a, i, float(got[2]), path)
            n_rec += 1
    return n_rec


@pytest.mark.parametrize('scenario,auto_reset,ticks', [('stage1', 1, 300), ('circle', 0, 150)])
def test_tracker_against_oracle(built, scenario, auto_reset, ticks):
    from rl_collision_avoidance_b200.evaluation import EpisodeTracker
    # circle: 16 robots on a 4 m circle meet at the centre within the run and collide
    sc = make_scenario('stage1') if scenario == 'stage1' else make_scenario('circle', robots_per_world=16, radius=4.0)
    env, orc = _pair(sc, worlds=2, auto_reset=auto_reset, seed=11)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    E = 4
    tr = EpisodeTracker(env, E)
    ref = _HostRecords(orc.N, env.cfg.dt, env.cfg.v_min, env.cfg.v_max)
    rng = np.random.default_rng(1)
    for t in range(ticks):
        a = random_actions(rng, orc.N)
        pose0, ep0 = orc.pose.copy(), orc.meta[:, 1].copy()
        env.control_vel(torch.from_numpy(a).cuda())
        tr.track()
        orc.step(a)
        ref.tick(pose0, ep0, a, orc.pose, orc.flags, orc.eplog)
    assert_state_equal(env, orc, scenario)
    n_rec = _check_records(tr, ref, E)
    assert n_rec > 10
    results = {r[0] for rows in ref.rec for r in rows}
    assert results <= {1, 2, 3} and (2 in results or 3 in results), results
    if auto_reset == 0:                                     # one episode: at most the first termination
        assert max(len(rows) for rows in ref.rec) == 1
    # open agents: in an episode that has not ended
    expect_open = ref.closed != orc.meta[:, 1]
    assert np.array_equal(tr.open.cpu().numpy() != 0, expect_open)


def test_stage2_records_only_the_first_end(built):
    """auto_reset=2: a finished robot idles (done = 1, result 0) until its group re-spawns; those ticks add nothing."""
    from rl_collision_avoidance_b200.evaluation import EpisodeTracker
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage2', num_worlds=2, seed=13, auto_reset=2)
    env.reset_pose()
    tr = EpisodeTracker(env, 8)
    rng = np.random.default_rng(2)
    prev = tr.count.clone()
    idle_ticks = resets = 0
    for t in range(420):
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda())
        tr.track()
        fl = env.flags.clone()
        cnt = tr.count.clone()
        ended = fl[:, 2] != 0
        assert torch.equal(cnt - prev, ended.int()), t
        rec = tr.records[torch.arange(env.N, device='cuda'), (cnt - 1).clamp(0, 7).long()]
        ep = env.eplog
        kept = ended & (cnt <= 8)
        assert torch.equal(rec[kept, 0], ep[kept, 6]) and torch.equal(rec[kept, 1], ep[kept, 3])
        idle_ticks += int(((fl[:, 0] != 0) & ~ended).sum())
        resets += int(fl[:, 3].sum())
        prev = cnt
    assert idle_ticks > 0 and resets > 0


def test_evaluate_stage1_three_episodes(built):
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage1', num_worlds=2, seed=3, auto_reset=1)
    pol = _policy('stage1_2.pth', env.N)
    out = evaluate(env, pol, 3, max_ticks=300, check_every=25)
    cnt = out['tracker'].count.cpu().numpy()
    p = out['totals']
    assert p[0] + p[1] + p[2] == np.minimum(cnt, 3).sum()
    assert p[3] == (cnt < 3).sum()                           # every robot short of 3 records is in an episode
    assert np.all((cnt >= 3) | (out['ticks'] == 300))
    recs = out['tracker'].records.cpu().numpy()
    assert set(np.unique(recs[cnt >= 3][:, :, 0])) <= {1.0, 2.0, 3.0}
    assert out['metrics']['reached'] > 0


def test_evaluate_is_deterministic_and_shard_invariant(built):
    """8 stage-1 worlds in one handle, and as two handles (world_offset 0 and 4): bit-identical per-world partials and
    totals; the same evaluation twice gives the same bits."""
    from rl_collision_avoidance_b200.evaluation import evaluate, totals
    from rl_collision_avoidance_b200.stage_world import StageWorld
    pol = _policy('stage1_2.pth', 8 * 24)
    env = StageWorld(512, scenario='stage1', num_worlds=8, seed=5, auto_reset=1)
    a = evaluate(env, pol, 2, max_ticks=320)
    b = evaluate(env, pol, 2, max_ticks=320)
    assert np.array_equal(a['partials'], b['partials']) and np.array_equal(a['totals'], b['totals'])
    del env
    parts = []
    for off in (0, 4):
        e = StageWorld(512, scenario='stage1', num_worlds=4, seed=5, auto_reset=1, world_offset=off)
        parts.append(evaluate(e, pol, 2, max_ticks=320)['partials'])
    sharded = np.concatenate(parts)
    assert np.array_equal(sharded.view(np.uint64), a['partials'].view(np.uint64))
    assert np.array_equal(totals(sharded).view(np.uint64), a['totals'].view(np.uint64))
    assert a['totals'][0] > 0


def test_reduce_matches_host_code(built):
    """rlca_eval_reduce on the device and rlca_eval_reduce_host on the records it read: the same bits."""
    from rl_collision_avoidance_b200.evaluation import evaluate, reduce_host
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario='stage2', num_worlds=3, seed=2, auto_reset=2)
    out = evaluate(env, _policy('stage2.pth', env.N), 2, max_ticks=402)
    tr = out['tracker']
    host = reduce_host(env.cfg, tr.records.cpu().numpy(), tr.count.cpu().numpy(), tr.open.cpu().numpy())
    assert np.array_equal(host.view(np.uint64), out['partials'].view(np.uint64))
    assert np.array_equal(tr.partials(1, 2), out['partials'][1:3])


def test_circle_evaluate_matches_circle_test(built):
    """Circle, stage2.pth, 2 worlds, 50 ticks: the recorded result codes and ticks are circle_test.enjoy's first
    terminations on the same seed."""
    sys.path.insert(0, ROOT)
    import circle_test
    from rl_collision_avoidance_b200.circle_world import StageWorld
    from rl_collision_avoidance_b200.evaluation import evaluate
    env = StageWorld(512, num_worlds=2, seed=4, auto_reset=0)
    pol = _policy('stage2.pth', env.N)
    ever, result, steps_to_end, steps = circle_test.enjoy(env, pol, [[0, -1], [1, 1]], 50)
    ever, result, steps_to_end = ever.cpu().numpy(), result.cpu().numpy(), steps_to_end.cpu().numpy()
    env2 = StageWorld(512, num_worlds=2, seed=4, auto_reset=0)
    out = evaluate(env2, pol, 1, max_ticks=steps, check_every=steps)
    tr = out['tracker']
    cnt = tr.count.cpu().numpy()
    rec = tr.records.cpu().numpy()[:, 0]
    assert np.array_equal(cnt, ever.astype(np.int32))
    assert np.array_equal(rec[ever, 0].astype(np.uint8), result[ever])
    assert np.array_equal(rec[ever, 1].astype(np.int32), steps_to_end[ever])
    assert out['totals'][3] == (~ever).sum()


@pytest.mark.parametrize('K,r,worlds', [(12, 10.0, 2), (64, 25.0, 1)])
def test_circle_k_robots_parity(built, K, r, worlds):
    """K robots on the circle (auto_reset=1: the circle tables re-spawn too): GPU state bit-equal to the oracle."""
    sc = make_scenario('circle', robots_per_world=K, radius=r)
    env, orc = _pair(sc, worlds=worlds, auto_reset=1, seed=9)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    assert_state_equal(env, orc, 'reset')
    rng = np.random.default_rng(K)
    for t in range(300):
        a = random_actions(rng, orc.N)
        env.control_vel(torch.from_numpy(a).cuda())
        orc.step(a)
        if t % 50 == 49:
            assert_state_equal(env, orc, f'tick {t}')
    assert_outputs_equal(env, orc, 'final')
    assert np.array_equal(env.flags.cpu().numpy(), orc.flags)
