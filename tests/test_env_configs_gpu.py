"""GPU parity across the configuration domain the C ABI accepts, not only the shipped configurations.

check_cfg takes 1..64 robots per world, any even beam count >= 2 with raw_beams >= beams, and any spawn budget
max_reject >= 1, and the kernels branch on exactly these values: the second re-spawn ballot word (R > 32), a last lidar
CTA with fewer than 4 viewers (R % 4), partial warps in the outline emitter (4R % 32), several re-spawns per warp
(> 8 in one world in one tick), the quad / aligned scalar / unaligned scalar beam passes (beams % 128, beams % 32,
buffer alignment) and the warp-wide rejection sampler around 32 and 64 tries.  Every case here compares the tick, the
observation and the raycast with the CPU oracle bit for bit (DESIGN.md §4), and asserts that the branch it is meant to
reach was taken: a parity test that never re-spawns a robot proves nothing about the re-spawn path.  Each case prints
its coverage counters (run with -s to see them)."""
import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, make_pair, random_actions

pytestmark = pytest.mark.gpu


def _check_tick(env, orc, tag, obs=None):
    """State, scan, local goal, reward, flags and the episode log of the agents that finished, bit for bit."""
    assert_state_equal(env, orc, tag)
    assert_outputs_equal(env, orc, tag, obs=obs)
    assert np.array_equal(env.reward.cpu().numpy().view(np.uint32), orc.reward.view(np.uint32)), f'{tag}: reward'
    assert np.array_equal(env.flags.cpu().numpy(), orc.flags), f'{tag}: flags'
    done = orc.flags[:, 0] != 0
    assert np.array_equal(env.eplog.cpu().numpy()[done].view(np.uint32), orc.eplog[done].view(np.uint32)), f'{tag}: eplog'


def _tick(env, orc, a, tag, **kw):
    env.control_vel(torch.from_numpy(a).cuda(), **kw)
    orc.step(a)
    _check_tick(env, orc, tag, obs=kw.get('obs_out'))


def _start(env, orc):
    """reset_world, then reset_pose (spawn sampler + observe), both against the oracle."""
    orc.reset_world()
    assert_state_equal(env, orc, 'reset_world')
    env.reset_pose()
    orc.reset_pose()
    assert_state_equal(env, orc, 'reset_pose')
    assert_outputs_equal(env, orc, 'reset_pose observation')


def _check_raycast(env, orc, rng, half, tag):
    """Stand-alone sweep from random poses inside +-half metres (and one far outside the map), normalised and raw."""
    pose = np.zeros((orc.N, 4), np.float32)
    pose[:, 0] = rng.uniform(-half, half, orc.N)
    pose[:, 1] = rng.uniform(-half, half, orc.N)
    pose[:, 2] = rng.uniform(-np.pi, np.pi, orc.N)
    pose[-1, :2] = [half + 50.0, 0.0]
    for normalise in (False, True):
        got = env.raycast(torch.from_numpy(pose).cuda(), normalise=normalise).cpu().numpy()
        ref = orc.raycast(pose, normalise=normalise)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), \
            f'{tag} raycast normalise={normalise}: {np.argwhere(got.view(np.uint32) != ref.view(np.uint32))[:4]}'


# ---------------------------------------------------------------- robots per world, stage-1 map
@pytest.mark.parametrize('R', [1, 2, 3, 5, 31, 32, 33, 63, 64])
def test_stage1_robot_counts(built, R):
    worlds = 3 if R <= 5 else 2
    sc, env, orc = make_pair('stage1', num_worlds=worlds, auto_reset=1, seed=1, robots_per_world=R)
    _start(env, orc)
    rng = np.random.default_rng(1)
    respawns = high = busiest = 0
    for t in range(120):
        _tick(env, orc, random_actions(rng, orc.N, wide=True), f'R={R} tick {t}')
        rs = orc.flags[:, 3].reshape(worlds, R) != 0
        respawns += int(rs.sum())
        high += int(rs[:, 32:].sum())
        busiest = max(busiest, int(rs.sum(1).max()))
    # observe from the moved poses, a goal for them, and a stand-alone sweep
    mask = (np.arange(orc.N) % 2 == 0).astype(np.uint8)
    env.generate_goal_point(torch.from_numpy(mask))
    orc.generate_goal_point(mask)
    assert_state_equal(env, orc, f'R={R} generate_goal_point')
    assert_outputs_equal(env, orc, f'R={R} generate_goal_point observation')
    _check_raycast(env, orc, rng, 9.0, f'R={R}')
    print(f'\n[robots R={R} x {worlds} worlds] re-spawns {respawns}, of robots >= 32: {high}, '
          f'most in one world in one tick: {busiest}')
    assert respawns > 0
    if R > 32:
        assert high > 0, 'no robot of the second ballot word re-spawned'
    if R >= 63:
        assert busiest > 8, 'no warp ran two re-spawns in one tick'


def test_stage1_mass_time_out(built):
    """64 robots, zero commands until the stage-1 time-out: nobody moves, crashes or arrives, so all 64 robots of every
    world time out on the same tick and re-spawn together - every warp of the physics CTA runs 8 spawns."""
    R, worlds = 64, 2
    sc, env, orc = make_pair('stage1', num_worlds=worlds, auto_reset=1, seed=4, robots_per_world=R)
    _start(env, orc)
    zero = np.zeros((orc.N, 2), np.float32)
    mass_tick = None
    for t in range(sc.timeout + 3):
        _tick(env, orc, zero, f'tick {t}')
        n = int(orc.flags[:, 3].sum())
        if n:
            assert mass_tick is None and n == orc.N, (t, n)
            assert np.all(orc.flags[:, 2] == 3) and np.all(orc.flags[:, 0] == 1)      # all time-outs
            mass_tick = t
    print(f'\n[mass time-out R=64 x {worlds} worlds] all {orc.N} robots re-spawned on tick {mass_tick}')
    assert mass_tick == sc.timeout


# ---------------------------------------------------------------- robots per world, circle map (global-grid lidar)
@pytest.mark.parametrize('K,hint', [(7, 0), (33, 0), (7, 3), (33, 5)])
def test_circle_robot_counts(built, K, hint):
    sc, env, orc = make_pair('circle', num_worlds=2, auto_reset=1, seed=3, robots_per_world=K, ctas_per_world=hint)
    if hint:
        rpc = -(-K // hint)
        slices = -(-K // rpc)
        last = K - (slices - 1) * rpc
        assert 0 < last < rpc, (K, hint, rpc, last)                      # the last slice is ragged
        print(f'\n[circle K={K} hint {hint}] {slices} slices of {rpc} viewers, last {last}')
    _start(env, orc)
    rng = np.random.default_rng(6)
    for t in range(8):
        a = random_actions(rng, orc.N, wide=True)
        _tick(env, orc, a, f'K={K} tick {t}')
    _check_raycast(env, orc, rng, 29.0, f'K={K}')


# ---------------------------------------------------------------- beam counts, small-map lidar
SMALL_BEAMS = [(b, None) for b in (2, 4, 30, 32, 34, 64, 96, 130, 256, 510, 2048)] + \
              [(2, 2), (2, 721), (30, 30), (30, 721), (130, 130), (130, 721), (256, 721), (510, 721), (512, 721)]


def _beam_path(beams):
    return 'quad' if beams % 128 == 0 else 'aligned scalar' if beams % 32 == 0 else 'unaligned scalar'


@pytest.mark.parametrize('beams,raw', SMALL_BEAMS)
def test_small_map_beam_counts(built, beams, raw):
    """Tick, observe and raycast (normalised and raw) at beam counts of every beam-pass path, below one warp of beams
    included, with sub-sampling from an odd raw count and identity sub-sampling."""
    sc, env, orc = make_pair('stage1', num_worlds=2, beams=beams, raw_beams=raw, auto_reset=1, seed=5)
    assert orc.cfg.raw_beams == (raw or max(512, beams))
    print(f'\n[stage1 beams {beams} raw {orc.cfg.raw_beams}] {_beam_path(beams)} beam pass')
    _start(env, orc)
    rng = np.random.default_rng(beams)
    for t in range(30):
        _tick(env, orc, random_actions(rng, orc.N, wide=True), f'beams {beams} tick {t}')
    env.generate_goal_point()
    orc.generate_goal_point()
    assert_outputs_equal(env, orc, f'beams {beams} observe')
    _check_raycast(env, orc, rng, 9.0, f'beams {beams}')
    assert (orc.obs < 0.49).any() and (orc.obs > 0.49).any()          # hits and misses


# ---------------------------------------------------------------- beam counts, big-map lidar
@pytest.mark.parametrize('beams', [2, 30, 180])
def test_big_map_beam_counts(built, beams):
    sc, env, orc = make_pair('circle', num_worlds=2, beams=beams, auto_reset=1, seed=7)
    _start(env, orc)
    rng = np.random.default_rng(beams)
    for t in range(4):
        a = random_actions(rng, orc.N)
        a[:, 0] = 1.0
        _tick(env, orc, a, f'circle beams {beams} tick {t}')
    _check_raycast(env, orc, rng, 29.0, f'circle beams {beams}')


# ---------------------------------------------------------------- scan FIFO on every store path
def _misaligned(shape):
    """A float32 CUDA tensor that starts one float past a 16-byte boundary."""
    n = int(np.prod(shape))
    t = torch.empty(n + 4, device='cuda')
    base = (16 - t.data_ptr() % 16) % 16 // 4
    return t[base + 1:base + 1 + n].view(*shape)


FIFO_CASES = [('stage1', 512, False), ('stage1', 96, False), ('stage1', 512, True), ('stage1', 180, False),
              ('circle', 180, False)]


@pytest.mark.parametrize('scenario,beams,misaligned', FIFO_CASES,
                         ids=['quad-512', 'aligned-96', 'aligned-512-offset', 'unaligned-180', 'circle-180'])
def test_scan_fifo_store_paths(built, scenario, beams, misaligned):
    """stack_out = [stack_in[1], stack_in[2], scan], three copies of the scan for a robot re-spawned this tick (the deque
    of ppo_stage1.py:60,87-89), on the quad, aligned scalar, unaligned scalar and big-map store paths."""
    if scenario == 'circle':           # 12 robots on a 3 m circle driving inwards: they meet and re-spawn within 20 ticks
        sc, env, orc = make_pair('circle', num_worlds=2, beams=beams, auto_reset=1, seed=3, robots_per_world=12,
                                 radius=3.0)
        ticks = 40
    else:
        sc, env, orc = make_pair('stage1', num_worlds=3, beams=beams, auto_reset=1, seed=5)
        ticks = 60
    _start(env, orc)
    N = orc.N
    ref = np.repeat(orc.obs[:, None, :], 3, axis=1).copy()
    make = _misaligned if misaligned else (lambda shape: torch.empty(*shape, device='cuda'))
    stacks = [make((N, 3, beams)), make((N, 3, beams))]
    stacks[0].copy_(torch.from_numpy(ref))
    obs_out = make((N, beams)) if misaligned else None
    if misaligned:
        assert all(t.data_ptr() % 16 == 4 for t in (stacks[0], stacks[1], obs_out))
    rng = np.random.default_rng(2)
    respawned = 0
    for t in range(ticks):
        a = random_actions(rng, N, wide=scenario == 'stage1')
        if scenario == 'circle':
            a[:, 0] = 1.0
            a[:, 1] *= 0.3
        _tick(env, orc, a, f'tick {t}', obs_out=obs_out, stack_in=stacks[t % 2], stack_out=stacks[(t + 1) % 2])
        ref = np.stack([ref[:, 1], ref[:, 2], orc.obs], 1)
        rs = orc.flags[:, 3] != 0
        ref[rs] = orc.obs[rs][:, None, :]
        respawned += int(rs.sum())
        got = stacks[(t + 1) % 2].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), f'FIFO tick {t}: rows ' \
            f'{np.unique(np.nonzero(got != ref)[0])[:8]}'
    print(f'\n[FIFO {scenario} {beams} beams{" misaligned" if misaligned else ""}] '
          f'{_beam_path(beams) if scenario == "stage1" else "big-map"} store path, {respawned} re-spawned rows')
    assert respawned > 0


@pytest.mark.parametrize('zero_copy', [0, 1, 2])
@pytest.mark.parametrize('beams', [96, 180])
def test_step_host_mirror_scalar_paths(built, beams, zero_copy):
    """step_host with the scalar beam passes (no quads): the host mirror / copies equal the device outputs and the
    oracle, in world ranges (3 chunks over 4 worlds)."""
    sc, env, orc = make_pair('stage1', num_worlds=4, beams=beams, auto_reset=1, seed=2)
    env.set_host_chunks(3)
    env.set_host_zero_copy(zero_copy)
    _start(env, orc)
    rng = np.random.default_rng(3)
    a_host = torch.empty(orc.N, 2).pin_memory()
    respawns = 0
    for t in range(30):
        a = random_actions(rng, orc.N, wide=True)
        a_host.copy_(torch.from_numpy(a))
        h = env.step_host(a_host)
        orc.step(a)
        assert np.array_equal(h['obs'].numpy().view(np.uint32), orc.obs.view(np.uint32)), f'host obs tick {t}'
        assert np.array_equal(h['reward'].numpy().view(np.uint32), orc.reward.view(np.uint32)), f'host reward tick {t}'
        assert np.array_equal(h['flags'].numpy(), orc.flags), f'host flags tick {t}'
        assert np.array_equal(h['gs'].numpy().view(np.uint32), orc.gs.view(np.uint32)), f'host gs tick {t}'
        _check_tick(env, orc, f'step_host device outputs tick {t}')
        respawns += int(orc.flags[:, 3].sum())
    assert respawns > 0


# ---------------------------------------------------------------- spawn budget
def _exhausted(scenario, sc, worlds, prev, pose, goal):
    """(spawns, goals) that no try accepted, so the sampler took its last try: a stage-1 spawn outside the 9 m disc or
    a goal outside the disc or the 8-10 m ring round its spawn; a stage-2 spawn (random rows) nearer than 7 m to the
    pose it left or a goal (random rows) nearer than 7 m to its spawn.  1e-4 m margins keep float rounding out."""
    x, y = pose[:, 0].astype(np.float64), pose[:, 1].astype(np.float64)
    gx, gy = goal[:, 0].astype(np.float64), goal[:, 1].astype(np.float64)
    dg = np.hypot(gx - x, gy - y)
    if scenario == 'stage1':
        sp = np.hypot(x, y) > 9.0 + 1e-4
        gl = (np.hypot(gx, gy) > 9.0 + 1e-4) | (dg > 10.0 + 1e-4) | (dg < 8.0 - 1e-4)
        return sp, gl
    sp = np.tile(sc.init_tab[:, 3] != 0, worlds) & (np.hypot(x - prev[:, 0], y - prev[:, 1]) < 7.0 - 1e-4)
    gl = np.tile(sc.goal_tab[:, 2] != 0, worlds) & (dg < 7.0 - 1e-4)
    return sp, gl


@pytest.mark.parametrize('max_reject', [1, 2, 31, 32, 33, 64, 65])
@pytest.mark.parametrize('scenario,auto_reset', [('stage1', 1), ('stage2', 1), ('stage2', 2)])
def test_spawn_budget(built, scenario, auto_reset, max_reject):
    """Rejection sampling with a budget of 1 .. 65 tries: reset_pose (repeatedly, many agents), generate_goal_point
    and the tick's re-spawns.  Where the budget can run out, it must have run out somewhere."""
    # ticks: re-spawns inside the physics launch
    sc, env, orc = make_pair(scenario, num_worlds=3, auto_reset=auto_reset, seed=3, max_reject=max_reject)
    _start(env, orc)
    rng = np.random.default_rng(1)
    respawns = tick_goals = 0
    for t in range(80):
        _tick(env, orc, random_actions(rng, orc.N, wide=True), f'max_reject {max_reject} tick {t}')
        rs = orc.flags[:, 3] != 0
        respawns += int(rs.sum())
        tick_goals += int((_exhausted(scenario, sc, 3, orc.pose, orc.pose, orc.goal)[1] & rs).sum())
    mask = (np.arange(orc.N) % 3 != 0).astype(np.uint8)
    env.generate_goal_point(torch.from_numpy(mask))
    orc.generate_goal_point(mask)
    assert_state_equal(env, orc, 'generate_goal_point')
    assert_outputs_equal(env, orc, 'generate_goal_point observation')
    assert respawns > 0
    # reset_pose: a batch of agents, several episodes each
    worlds = 40 if scenario == 'stage1' else 24
    sc, env, orc = make_pair(scenario, num_worlds=worlds, auto_reset=auto_reset, seed=3, max_reject=max_reject)
    orc.reset_world()
    spawns = goals = 0
    for k in range(5):
        prev = orc.pose.copy()
        env.reset_pose()
        orc.reset_pose()
        assert_state_equal(env, orc, f'reset_pose {k}')
        assert_outputs_equal(env, orc, f'reset_pose {k} observation')
        sp, gl = _exhausted(scenario, sc, worlds, prev, orc.pose, orc.goal)
        spawns += int(sp.sum())
        goals += int(gl.sum())
    env.generate_goal_point()
    orc.generate_goal_point()
    assert_state_equal(env, orc, 'generate_goal_point after reset_pose')
    print(f'\n[{scenario} auto_reset={auto_reset} max_reject={max_reject}] tick re-spawns {respawns}, exhausted goals '
          f'in ticks {tick_goals}; reset_pose exhausted spawns {spawns}, goals {goals} of {5 * orc.N}')
    if max_reject <= 2:
        assert spawns > 0 and goals > 0
    if scenario == 'stage1' and max_reject == 33:
        assert goals > 0, 'no goal search ran out in the group of tries from 32'
