"""GPU parity: the fused CUDA tick (through the C ABI) vs the CPU oracle, bit for bit.

The numerics contract (DESIGN.md §4) makes poses, ranges, rewards and flags exactly
reproducible, so every comparison here is np.array_equal on the raw bits — tighter than
the north-star's 1e-4 fp32 tolerance (collision flags bit-exact)."""
import math

import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, make_pair, random_actions

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('scenario,worlds', [('stage1', 5), ('stage2', 3)])
def test_reset_and_observe_match_oracle(built, scenario, worlds):
    sc, env, orc = make_pair(scenario, num_worlds=worlds)
    orc.reset_world()
    assert_state_equal(env, orc, 'after reset_world')
    env.reset_pose()
    orc.reset_pose()
    assert_state_equal(env, orc, 'after reset_pose')
    assert_outputs_equal(env, orc, 'first observation')


@pytest.mark.parametrize('scenario,worlds,beams', [('stage1', 5, 512), ('stage2', 2, 512), ('stage1', 2, 180)])
def test_rollout_bit_exact(built, scenario, worlds, beams):
    sc, env, orc = make_pair(scenario, num_worlds=worlds, beams=beams, auto_reset=True, seed=7)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(1)
    seen = np.zeros(4, int)
    for t in range(260):
        a = random_actions(rng, orc.N, wide=True)
        if t % 37 == 5:
            a[::7] = 0.0          # exact-zero command: move (and stall update) skipped
        if t == 11:
            a[3] = [np.nan, np.inf]
        env.control_vel(torch.from_numpy(a).cuda())
        orc.step(a)
        assert_state_equal(env, orc, f'tick {t}')
        assert_outputs_equal(env, orc, f'tick {t}')
        torch.cuda.synchronize()
        assert np.array_equal(env.reward.cpu().numpy().view(np.uint32), orc.reward.view(np.uint32)), f'reward tick {t}'
        assert np.array_equal(env.flags.cpu().numpy(), orc.flags), f'flags tick {t}'
        done = orc.flags[:, 0] != 0
        assert np.array_equal(env.eplog.cpu().numpy()[done], orc.eplog[done]), f'eplog tick {t}'
        for k in range(4):
            seen[k] += int((orc.flags[:, 2] == k).sum())
    # the rollout must actually have exercised crashes, time-outs (stage1: 150) and re-spawns
    assert seen[2] > 0 and seen[3] > 0, seen


def test_manual_reset_and_live_mask(built):
    """Stage-2 style group-synchronous episodes: no auto reset, finished agents idle on their
    last command with live=0 (ppo_stage2.py:72-84), then a masked reset_pose."""
    sc, env, orc = make_pair('stage2', num_worlds=2, auto_reset=False, seed=3)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(5)
    live = np.ones(orc.N, np.uint8)
    for t in range(120):
        a = random_actions(rng, orc.N)
        env.control_vel(torch.from_numpy(a).cuda(), live=torch.from_numpy(live).cuda())
        orc.step(a, live=live)
        assert_state_equal(env, orc, f'tick {t}')
        assert_outputs_equal(env, orc, f'tick {t}')
        assert np.array_equal(env.flags.cpu().numpy(), orc.flags)
        assert np.array_equal(env.reward.cpu().numpy().view(np.uint32), orc.reward.view(np.uint32))
        live[orc.flags[:, 0] != 0] = 0
        if t == 80:
            mask = (live == 0).astype(np.uint8)
            assert mask.sum() > 0
            env.reset_pose(torch.from_numpy(mask).cuda())
            orc.reset_pose(mask)
            live[:] = 1
            assert_state_equal(env, orc, 'masked reset')
            assert_outputs_equal(env, orc, 'masked reset')


def test_ctas_per_world_invariance(built):
    """The launch shape hint must not change any result (small maps: fixed 4 robots per lidar CTA, the hint is ignored;
    the big-map lidar honours it - see test_circle_launch_shape_invariance)."""
    outs = []
    for s in (1, 3, 8):
        sc, env, orc = make_pair('stage1', num_worlds=4, seed=11, ctas_per_world=s)
        env.reset_pose()
        rng = np.random.default_rng(2)
        for t in range(40):
            env.control_vel(torch.from_numpy(random_actions(rng, orc.N)).cuda())
        torch.cuda.synchronize()
        outs.append((env.obs.cpu().numpy().copy(), env.state['pose'].cpu().numpy().copy(),
                     env.reward.cpu().numpy().copy(), env.flags.cpu().numpy().copy()))
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert np.array_equal(a, b)


@pytest.mark.parametrize('scenario', ['stage1', 'stage2'])
def test_standalone_raycast_matches_oracle(built, scenario):
    sc, env, orc = make_pair(scenario, num_worlds=6, seed=1)
    rng = np.random.default_rng(9)
    half = 9.0 if scenario == 'stage1' else 19.0
    pose = np.zeros((orc.N, 4), np.float32)
    pose[:, 0] = rng.uniform(-half, half, orc.N)
    pose[:, 1] = rng.uniform(-half, half, orc.N)
    pose[:, 2] = rng.uniform(-np.pi, np.pi, orc.N)
    pose[5, :2] = [half + 50.0, 0.0]       # a robot far outside the map: every beam misses
    for normalise in (False, True):
        got = env.raycast(torch.from_numpy(pose).cuda(), normalise=normalise).cpu().numpy()
        ref = orc.raycast(pose, normalise=normalise)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), np.abs(got - ref).max()
    raw = orc.raycast(pose)
    assert raw.min() >= 0.0 and raw.max() <= 6.0 + 1e-5
    assert np.all(raw[5] == 6.0)


def test_headline_size_properties(built):
    """BASELINE headline size (171 worlds x 24 robots x 512 beams): size-independent properties.
    (1) determinism, (2) world independence: world w of the big batch equals the same world run
    alone with the matching global world offset, checked against the oracle for a few worlds."""
    worlds = 171
    sc, env, _ = make_pair('stage1', num_worlds=worlds, seed=0, gpu=True)
    env.reset_pose()
    rng = np.random.default_rng(4)
    acts = [random_actions(rng, env.N) for _ in range(30)]
    for a in acts:
        env.control_vel(torch.from_numpy(a).cuda())
    torch.cuda.synchronize()
    obs_big = env.obs.cpu().numpy()
    pose_big = env.state['pose'].cpu().numpy()
    assert obs_big.min() >= -0.5 and obs_big.max() <= 0.5 + 1e-6
    # same thing again -> identical
    sc2, env2, _ = make_pair('stage1', num_worlds=worlds, seed=0)
    env2.reset_pose()
    for a in acts:
        env2.control_vel(torch.from_numpy(a).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(env2.obs.cpu().numpy(), obs_big)
    # worlds 100..102 alone on the oracle with world_offset=100
    R = 24
    _, _, orc = make_pair('stage1', num_worlds=3, seed=0, world_offset=100, gpu=False)
    orc.reset_world()
    orc.reset_pose()
    for a in acts:
        orc.step(a[100 * R:103 * R])
    assert np.array_equal(orc.obs.view(np.uint32), obs_big[100 * R:103 * R].view(np.uint32))
    assert np.array_equal(orc.pose.view(np.uint32), pose_big[100 * R:103 * R].view(np.uint32))


@pytest.mark.parametrize('zero_copy', [0, 1, 2])
@pytest.mark.parametrize('scenario,worlds,chunks', [('stage1', 4, 0), ('stage1', 7, 3), ('stage1', 3, 16),
                                                    ('stage1', 5, 1), ('stage2', 5, 2)])
def test_step_host_matches_device_path(built, scenario, worlds, chunks, zero_copy):
    """The host-buffer call, serial (1) and pipelined over world ranges (uneven ranges, more chunks than worlds,
    the stage-2 group barrier inside a range), with DMA copies or with the kernel reading actions from / mirroring the
    small outputs to mapped host memory: bit-identical to the oracle, i.e. to the single launch."""
    sc, env, orc = make_pair(scenario, num_worlds=worlds, seed=2, auto_reset=2 if scenario == 'stage2' else True)
    env.set_host_chunks(chunks)
    env.set_host_zero_copy(zero_copy)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(3)
    a_host = torch.empty(orc.N, 2).pin_memory()
    for t in range(20):
        a = random_actions(rng, orc.N)
        a_host.copy_(torch.from_numpy(a))
        h = env.step_host(a_host)
        orc.step(a)
        assert np.array_equal(h['obs'].numpy().view(np.uint32), orc.obs.view(np.uint32))
        assert np.array_equal(h['reward'].numpy().view(np.uint32), orc.reward.view(np.uint32))
        assert np.array_equal(h['flags'].numpy(), orc.flags)
        assert np.array_equal(h['gs'].numpy().view(np.uint32), orc.gs.view(np.uint32))
        assert_outputs_equal(env, orc, f'device copies, step_host t={t}')      # io's device buffers are written too
    assert_state_equal(env, orc, f'step_host chunks={chunks}')


def test_step_host_with_pageable_buffers_falls_back_to_copies(built):
    sc, env, orc = make_pair('stage1', num_worlds=3, seed=4)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    env._host = dict(obs=torch.empty(env.N, 512), reward=torch.empty(env.N), flags=torch.empty(env.N, 4, dtype=torch.uint8),
                     gs=torch.empty(env.N, 4))                 # pageable: no device-mapped alias
    env._host_args = [(env._state_struct(k), env._state_struct(1 - k), env._io()) for k in (0, 1)]
    rng = np.random.default_rng(8)
    for t in range(5):
        a = random_actions(rng, orc.N)
        h = env.step_host(torch.from_numpy(a))
        orc.step(a)
        assert np.array_equal(h['obs'].numpy().view(np.uint32), orc.obs.view(np.uint32))
        assert np.array_equal(h['flags'].numpy(), orc.flags)


def test_errors_are_loud(built):
    import ctypes as C
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    cfg = _lib.EnvConfig()
    h = C.c_void_p()
    assert lib.rlca_env_create(C.byref(cfg), C.byref(h)) != 0      # empty config is invalid
    assert b'robots_per_world' in lib.rlca_last_error()
    sc, env, _ = make_pair('stage1', num_worlds=1)
    with pytest.raises(_lib.RlcaError):
        env.raycast(torch.zeros(env.N, 4), normalise=False, out=None) if False else _lib.check(
            lib.rlca_raycast(env._h, None, None, 0, None))


def test_group_synchronous_stage2_mode(built):
    """auto_reset=2: finished robots idle until their whole group is done, then the group re-spawns
    (ppo_stage2.py:72-84,105-106) — all inside the tick, bit-exact against the oracle."""
    sc, env, orc = make_pair('stage2', num_worlds=2, auto_reset=2, seed=13)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    rng = np.random.default_rng(21)
    resets = idle = 0
    for t in range(420):
        a = random_actions(rng, orc.N)
        env.control_vel(torch.from_numpy(a).cuda())
        orc.step(a)
        if t % 7 == 0 or t > 400:
            assert_state_equal(env, orc, f'tick {t}')
            assert_outputs_equal(env, orc, f'tick {t}')
            assert np.array_equal(env.flags.cpu().numpy(), orc.flags)
            assert np.array_equal(env.reward.cpu().numpy().view(np.uint32), orc.reward.view(np.uint32))
        resets += int(orc.flags[:, 3].sum())
        idle += int((orc.meta[:, 3] != 0).sum())
        # a group is re-spawned together: was_reset is constant inside every group
        wr = orc.flags[:, 3].reshape(2, 44)
        for a0, b0 in zip(sc.groups[:-1], sc.groups[1:]):
            assert np.all(wr[:, a0:b0] == wr[:, a0:a0 + 1])
    assert resets > 0 and idle > 0, (resets, idle)


def test_fused_scan_fifo(built):
    """stack_out = [stack_in[1], stack_in[2], scan] and three copies of the scan after a re-spawn
    (the deque of ppo_stage1.py:60,87-89), written by the tick kernel itself."""
    sc, env, orc = make_pair('stage1', num_worlds=3, auto_reset=1, seed=5)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    N, B = orc.N, 512
    ref = np.repeat(orc.obs[:, None, :], 3, axis=1).copy()
    stacks = [torch.from_numpy(ref).cuda(), torch.empty(N, 3, B, device='cuda')]
    rng = np.random.default_rng(2)
    saw_reset = False
    for t in range(200):
        a = random_actions(rng, N)
        env.control_vel(torch.from_numpy(a).cuda(), stack_in=stacks[t % 2], stack_out=stacks[(t + 1) % 2])
        orc.step(a)
        ref = np.stack([ref[:, 1], ref[:, 2], orc.obs], 1)
        rs = orc.flags[:, 3] != 0
        ref[rs] = orc.obs[rs][:, None, :]
        saw_reset |= bool(rs.any())
        if t % 9 == 0 or t == 199:
            assert np.array_equal(stacks[(t + 1) % 2].cpu().numpy(), ref), f'tick {t}'
    assert saw_reset


def test_circle_world_global_grid_path(built):
    """circle.world (60 x 60 m at 0.01 m = 6000 x 6000 cells, 50 robots, antipodal goals): no first-hit table at this
    size - the library walks the static map through a distance field and scatters the other robots' outlines through
    the inverse walk lists (rlca_big_lidar_kernel).  Same oracle, same bit-exact bar (reset, observe, ticks incl. the
    |w| > 0.7 penalty, raycast)."""
    sc, env, orc = make_pair('circle', num_worlds=2, auto_reset=1, seed=3)
    orc.reset_world()
    assert_state_equal(env, orc, 'reset_world')
    env.reset_pose()
    orc.reset_pose()
    assert_state_equal(env, orc, 'reset_pose')
    assert_outputs_equal(env, orc, 'first observation')
    rng = np.random.default_rng(6)
    for t in range(12):
        a = random_actions(rng, orc.N)
        a[:, 0] = 1.0 if t < 8 else a[:, 0]          # drive inwards so that robots meet
        env.control_vel(torch.from_numpy(a).cuda())
        orc.step(a)
        assert_state_equal(env, orc, f'tick {t}')
        assert_outputs_equal(env, orc, f'tick {t}')
        assert np.array_equal(env.flags.cpu().numpy(), orc.flags)
        assert np.array_equal(env.reward.cpu().numpy().view(np.uint32), orc.reward.view(np.uint32))
    assert (orc.reward < -2.0).any() or (np.abs(orc.reward) > 0).any()
    # robots see their neighbours on the circle (3.1 m apart): some beams must return < 6 m
    assert (orc.obs < 0.49).any()
    pose = orc.pose.copy()
    got = env.raycast(torch.from_numpy(pose).cuda()).cpu().numpy()
    ref = orc.raycast(pose)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_circle_raycast_walls_corners_outside(built):
    """The big-map lidar's static part on hand-placed poses: robots 5 cm to 6.5 m from a wall of circle.world at all
    headings (distance-field walks of 1 to many jumps; the start-cell distance comes from shared memory), in the four
    corners, ON the wall cells, outside the floor plan (no distance field there: the walk reads the template), and
    pairs close enough for the long inverse lists of the scatter.  Scans must equal the cell-marching oracle's."""
    sc, env, orc = make_pair('circle', num_worlds=2, auto_reset=1, seed=5)
    orc.reset_world()
    env.reset_pose()
    orc.reset_pose()
    rng = np.random.default_rng(12)
    N = orc.N
    pose = orc.pose.copy()
    k = 0
    for d in (0.05, 0.11, 0.3, 0.8, 1.7, 3.0, 4.4, 5.9, 6.05, 6.5):          # distance to the wall at x = +30 / y = -30
        pose[k, :3] = (30.0 - d, rng.uniform(-20, 20), rng.uniform(-np.pi, np.pi)); k += 1
        pose[k, :3] = (rng.uniform(-20, 20), -30.0 + d, rng.uniform(-np.pi, np.pi)); k += 1
    for sx in (-1, 1):
        for sy in (-1, 1):                                                   # corners, 0.4 m and 3 m inside
            pose[k, :3] = (sx * 29.6, sy * 29.6, rng.uniform(-np.pi, np.pi)); k += 1
            pose[k, :3] = (sx * 27.0, sy * 27.0, math.atan2(sy, sx)); k += 1
    for x, y in ((30.0, 0.0), (-30.005, 3.0), (31.0, 0.0), (-36.5, -2.0), (0.0, 33.0), (29.0, 40.0)):   # on / beyond the walls
        pose[k, :3] = (x, y, rng.uniform(-np.pi, np.pi)); k += 1
    for i in range(6):                                                       # tight cluster: cells next to the viewer
        pose[k, :3] = (10.0 + 0.45 * (i % 3), -4.0 + 0.5 * (i // 3), rng.uniform(-np.pi, np.pi)); k += 1
    assert k <= 50
    pose[50:, :3] = pose[:50, :3]                                            # second world: same places, other headings
    pose[50:, 2] = rng.uniform(-np.pi, np.pi, 50)
    pose = pose.astype(np.float32)
    got = env.raycast(torch.from_numpy(pose).cuda()).cpu().numpy()
    ref = orc.raycast(pose)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), np.argwhere(got != ref)[:5]
    assert (ref < 5.99).mean() > 0.2 and (ref > 5.99).any()                  # walls and robots seen, and free beams too
    # the tick from those poses (collision against walls for the robots on / at them, re-spawns)
    env.control_pose(torch.from_numpy(pose[:, :3].copy()))
    orc.pose[:] = env.state['pose'].cpu().numpy()
    orc.observe()
    assert_outputs_equal(env, orc, 'scan after control_pose')
    a = random_actions(rng, N)
    env.control_vel(torch.from_numpy(a).cuda())
    orc.step(a)
    assert_outputs_equal(env, orc, 'tick from the hand-placed poses')


@pytest.mark.parametrize('scenario', ['stage1', 'stage2'])
def test_env_surface_leftovers(built, scenario):
    """generate_goal_point alone / generate_random_goal / generate_random_pose / control_pose / get_self_speedGT
    (stage_world1.py:119-120,171-177,237-274 and the stage-2 variants)."""
    sc, env, orc = make_pair(scenario, num_worlds=3, seed=17)
    env.reset_pose()
    orc.reset_world()
    orc.reset_pose()
    before = {k: v.clone() for k, v in env.state.items()}
    # the reference's call order reset_pose -> generate_goal_point re-derives the same goal: nothing changes
    env.generate_goal_point()
    orc.generate_goal_point()
    assert_state_equal(env, orc, 'generate_goal_point after reset_pose')
    for k, v in before.items():
        assert torch.equal(v, env.state[k]), k
    # the pose the NEXT reset_pose will use, without touching the state
    nxt = env.generate_random_pose().cpu().numpy()
    for k, v in before.items():
        assert torch.equal(v, env.state[k]), k
    # teleport two thirds of the robots, then a goal for where they are now
    rng = np.random.default_rng(3)
    new = np.stack([rng.uniform(-6, 6, orc.N), rng.uniform(-6, 6, orc.N), rng.uniform(-7, 7, orc.N)], 1).astype(np.float32)
    if scenario == 'stage2':
        new[:, 0] += 12.0
        new[:, 1] -= 8.0
    mask = (np.arange(orc.N) % 3 != 0)
    env.control_pose(torch.from_numpy(new), mask=torch.from_numpy(mask))
    th = np.float32(new[:, 2])
    got = env.state['pose'].cpu().numpy()
    assert np.array_equal(got[~mask], before['pose'].cpu().numpy()[~mask])
    assert np.allclose(got[mask, :2], new[mask, :2]) and np.all(np.abs(got[:, 2]) <= np.pi + 1e-6)
    assert np.allclose(np.cos(got[mask, 2]), np.cos(th[mask]), atol=1e-5) and np.allclose(np.sin(got[mask, 2]), np.sin(th[mask]), atol=1e-5)
    assert np.array_equal(env.state['meta'].cpu().numpy(), before['meta'].cpu().numpy())     # stall / counters untouched
    orc.pose[:] = got                                         # same poses on the oracle side, then compare the scans
    orc.observe()
    assert_outputs_equal(env, orc, 'scan after control_pose')
    want_goal = env.generate_random_goal().cpu().numpy()
    env.generate_goal_point(mask=torch.from_numpy(mask))
    orc.generate_goal_point(mask.astype(np.uint8))
    assert_state_equal(env, orc, 'generate_goal_point for the teleported robots')
    assert_outputs_equal(env, orc, 'local goal after generate_goal_point')
    assert np.array_equal(env.state['goal'].cpu().numpy()[mask, :2], want_goal[mask])
    if scenario == 'stage1':
        d = np.hypot(*(env.state['goal'].cpu().numpy()[mask, :2] - got[mask, :2]).T)
        assert np.all((d >= 8.0 - 1e-4) & (d <= 10.0 + 1e-4))          # generate_random_goal's acceptance ring
    # ground-truth speed: zero before a tick, then |dpose| / dt
    assert float(env.get_self_speedGT().abs().max()) == 0.0
    prev = env.state['pose'].cpu().numpy().copy()
    a = random_actions(rng, orc.N)
    env.control_vel(torch.from_numpy(a).cuda())
    cur = env.state['pose'].cpu().numpy()
    gt = env.get_self_speedGT().cpu().numpy()
    dth = (cur[:, 2] - prev[:, 2] + np.pi) % (2 * np.pi) - np.pi
    assert np.allclose(gt[:, 0], np.hypot(cur[:, 0] - prev[:, 0], cur[:, 1] - prev[:, 1]) * 10, atol=1e-4)
    assert np.allclose(gt[:, 1], dth * 10, atol=1e-4)
    moved = (env.flags.cpu().numpy()[:, 1] == 0) & (env.flags.cpu().numpy()[:, 3] == 0)
    assert np.allclose(gt[moved, 0], np.clip(a[moved, 0], 0, 1), atol=2e-4)      # un-crashed robots move at the command
    # and the pose generate_random_pose announced is the one reset_pose uses
    env.control_pose(torch.from_numpy(before['pose'].cpu().numpy()[:, :3]))
    env._st[env._cur]['meta'].copy_(before['meta'])
    env.reset_pose()
    assert np.array_equal(env.state['pose'].cpu().numpy()[:, :3], nxt)


def test_config_limits_are_rejected(built):
    """range_cells >= 2048 would overflow the 12-bit fields of the lidar walk key, and max_reject < 1 leaves a spawn
    without a try to take: loud errors, not wrong ranges or poses."""
    import ctypes as C
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario
    lib = _lib.load()
    sc = make_scenario('stage1')
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=1, beams=512)
    cfg.range_cells = 2500.0
    h = C.c_void_p()
    assert lib.rlca_env_create(C.byref(cfg), C.byref(h)) != 0
    assert b'range_cells' in lib.rlca_last_error()
    # a spawn takes at least one rejection-sampling try
    cfg = fill_config(_lib.EnvConfig(), sc, num_worlds=1, beams=512)
    cfg.max_reject = 0
    assert lib.rlca_env_create(C.byref(cfg), C.byref(h)) != 0
    assert b'max_reject' in lib.rlca_last_error()


def test_circle_launch_shape_invariance(built):
    """Big-map lidar: viewers per CTA (ctas_per_world hint 50 / 25 / 10) must not change any scan."""
    outs = []
    for s in (50, 25, 10):
        sc, env, orc = make_pair('circle', num_worlds=2, seed=5, auto_reset=1, ctas_per_world=s)
        env.reset_pose()
        rng = np.random.default_rng(2)
        for t in range(6):
            env.control_vel(torch.from_numpy(random_actions(rng, orc.N)).cuda())
        torch.cuda.synchronize()
        outs.append((env.obs.cpu().numpy().copy(), env.state['pose'].cpu().numpy().copy(), env.flags.cpu().numpy().copy()))
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert np.array_equal(a, b)
