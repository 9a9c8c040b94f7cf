"""Arena layouts on the device (DESIGN.md §9v): rlca_layout_arena and rlca_layout_arena_respawn against their host twins
bit for bit (both picks, failure status included, after every tick of a rollout), the env on the generated map against
the CPU oracle after a layout and after re-layouts, evaluate() with the policy and the map-aware baselines, and
ppo_stage2.py --scenario arena / --mix with an arena component end to end."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, random_actions

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
STAGE2 = os.path.join(CKPT, 'stage2.pth')


def _scenario(K=8, T=64, pick=0, timeout=None, **kw):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    return make_scenario('arena', robots_per_world=K, arenas=T, pick=pick, timeout=timeout, **kw)


def _env(sc, W, seed=0, world_offset=0, auto_reset=0, max_reject=4096):
    from rl_collision_avoidance_b200.stage_world import StageWorld
    return StageWorld(512, scenario=sc, num_worlds=W, seed=seed, auto_reset=auto_reset, world_offset=world_offset,
                      max_reject=max_reject)


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _tsame(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _host(env, flags):
    torch.cuda.synchronize()
    st = env.state
    return (st['pose'].cpu().numpy(), st['goal'].cpu().numpy(), st['acc'].cpu().numpy(), st['meta'].cpu().numpy(),
            flags.cpu().numpy())


@pytest.mark.parametrize('pick', [0, 1])
@pytest.mark.parametrize('K,T,W,wo,max_reject', [(8, 64, 1024, 0, 4096), (16, 9, 300, 17, 4096),
                                                 (12, 4, 64, 0, 8)])
def test_layout_kernel_equals_host_twin(built, pick, K, T, W, wo, max_reject):
    """rlca_layout_arena on random rows equals rlca_layout_arena_host bit for bit, status included (with 8 tries some
    worlds fail and keep their rows)."""
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.scenarios import arena_layout_host
    sc = _scenario(K, T, pick)
    env = _env(sc, W, seed=K + T, world_offset=wo, max_reject=max_reject)
    rng = np.random.default_rng(pick)
    rows = [rng.standard_normal((env.N, 4)).astype(np.float32) for _ in range(3)]
    for k, r in zip(('pose', 'goal', 'acc'), rows):
        env.state[k].copy_(torch.from_numpy(r))
    status = torch.full((W,), -7, dtype=torch.int32, device='cuda')
    lay = sc.layout
    params = _lib.LayoutParams(lay.side, lay.separation, lay.min_travel)
    st = env._state_struct(env._cur)
    _lib.check(env.lib.rlca_layout_arena(C.byref(env.cfg), C.byref(params), C.byref(env._arena), pick, C.byref(st),
                                         C.c_void_p(status.data_ptr()), env._stream()))
    want = arena_layout_host(env.cfg, lay, *rows)
    got = _host(env, env.flags)[:3] + (status.cpu().numpy(),)
    for name, x, y in zip(('pose', 'goal', 'acc', 'status'), got, want):
        assert _same(x, y), name
    if max_reject == 8:
        assert want[3].any() and not want[3].all()
    else:
        assert not want[3].any()


def _steer(gs, noise):
    w = torch.clamp(2.0 * torch.atan2(gs[:, 1], gs[:, 0]) + noise[:, 1], -1.0, 1.0)
    return torch.stack((torch.clamp(1.0 - noise[:, 0].abs(), 0.0, 1.0), w), 1).contiguous()


class Driver:
    """The trainer's per-tick sequence: tick with `live` into the stack / gs / flags buffers, then relayout_finished."""

    def __init__(self, env, horizon):
        n, dev = env.N, env.device
        self.env = env
        self.stacks = torch.empty(horizon + 1, n, 3, 512, device=dev)
        self.gs = torch.empty(horizon + 1, n, 4, device=dev)
        self.flags = torch.zeros(horizon, n, 4, dtype=torch.uint8, device=dev)
        self.stacks[0] = env.obs[:, None, :]
        self.gs[0] = env.gs

    def tick(self, t, action):
        self.env.control_vel(action, live=self.env.live, stack_in=self.stacks[t], stack_out=self.stacks[t + 1],
                             out={'flags': self.flags[t], 'gs': self.gs[t + 1]})

    def relayout(self, t):
        self.env.relayout_finished(self.stacks[t + 1], out={'gs': self.gs[t + 1], 'flags': self.flags[t]})


def _started(sc, W, seed, world_offset=0):
    env = _env(sc, W, seed=seed, world_offset=world_offset)
    env.reset_world()
    env.random_layout()
    return env


@pytest.mark.parametrize('pick', [0, 1])
def test_respawn_kernel_equals_host_twin_after_every_tick(built, pick):
    """100 ticks of noisy goal-seeking actions on 512 worlds with a 25-tick time-out: after every tick the state, live,
    status and flags equal rlca_layout_arena_respawn_host applied to the tick's output, and re-laid rows of the stack
    are the new scan; every world is re-laid at least twice, with pick 1 in more than one arena."""
    from rl_collision_avoidance_b200.scenarios import arena_relayout_host
    K, W, T = 8, 512, 100
    sc = _scenario(K, 64, pick, timeout=25)
    env = _started(sc, W, seed=3 + pick)
    d = Driver(env, T)
    gen = torch.Generator(device='cuda').manual_seed(pick)
    relaid = np.zeros(W, np.int64)
    cells = {}
    for t in range(T):
        d.tick(t, _steer(d.gs[t], 0.5 * torch.randn(env.N, 2, device='cuda', generator=gen)))
        before = _host(env, d.flags[t])
        stack_tick = d.stacks[t + 1].clone()
        d.relayout(t)
        want = arena_relayout_host(env.cfg, sc.layout, *before)
        got = _host(env, d.flags[t]) + (env.live.cpu().numpy(), env._relayout_status.cpu().numpy())
        for name, x, y in zip(('pose', 'goal', 'acc', 'meta', 'flags', 'live', 'status'), got, want):
            assert _same(x, y), f'tick {t}: {name} differs'
        assert not want[6].any()
        r = torch.from_numpy(want[4][:, 3] != 0).cuda()
        assert _tsame(d.stacks[t + 1][r], env.obs[r][:, None, :].expand(-1, 3, -1)), f'tick {t}: refreshed stack'
        assert _tsame(d.stacks[t + 1][~r], stack_tick[~r]), f'tick {t}: other stack rows'
        per_world = want[4][:, 3].reshape(W, K).all(1)
        relaid += per_world
        for w in np.flatnonzero(per_world)[:4]:
            cells.setdefault(w, set()).add(int(np.floor(want[0][w * K, 0] / 10.4)))
    assert relaid.min() >= 2, relaid.min()
    if pick == 1:
        assert any(len(v) > 1 for v in cells.values())


def test_env_matches_oracle_after_layout_and_relayouts(built):
    """From the layout on, through re-layouts (the device's, and the host twin on the oracle's rows), 60 random-action
    ticks on the generated map equal the oracle in state, scan, local goal, flags and live mask."""
    from oracle.oracle import OracleWorld, OrcConfig
    from rl_collision_avoidance_b200.scenarios import arena_relayout_host, fill_config
    K, W = 8, 24
    sc = _scenario(K, 64, 1, timeout=15)
    env = _started(sc, W, seed=11)
    ocfg = fill_config(OrcConfig(), sc, num_worlds=W, beams=512, auto_reset=0, seed=11)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    torch.cuda.synchronize()
    for k in ('pose', 'goal', 'acc', 'meta'):
        getattr(orc, k)[...] = env.state[k].cpu().numpy()
    orc.observe()
    assert_outputs_equal(env, orc, 'layout')
    rng = np.random.default_rng(11)
    stack = torch.empty(env.N, 3, 512, device='cuda')
    relaid = 0
    for t in range(60):
        a = random_actions(rng, orc.N)
        live = env.live.cpu().numpy()
        env.control_vel(torch.from_numpy(a).cuda(), live=env.live)
        orc.step(a, live=live)
        assert_state_equal(env, orc, f'tick {t}')
        assert_outputs_equal(env, orc, f'tick {t}')
        assert np.array_equal(env.flags.cpu().numpy(), orc.flags), f'tick {t}: flags differ'
        flags = env.flags.clone()
        env.relayout_finished(stack, out={'flags': flags})
        p, g, ac, m, f, lv, s = arena_relayout_host(env.cfg, sc.layout, orc.pose, orc.goal, orc.acc, orc.meta,
                                                    orc.flags)
        orc.pose[...], orc.goal[...], orc.acc[...], orc.meta[...] = p, g, ac, m
        orc.observe()
        relaid += int(f[:, 3].sum())
        assert_state_equal(env, orc, f'relayout {t}')
        assert_outputs_equal(env, orc, f'relayout {t}')
        assert _same(env.live.cpu().numpy(), lv) and not s.any()
    assert relaid > 0


def test_arena_map_takes_the_small_map_path(built):
    """The generated map (about 44 MB of first-hit table) stays on the small-map lidar, which reports its CTAs per SM;
    the random scenario's circle.world is a big map, for which the library reports 0."""
    from rl_collision_avoidance_b200.arenas import big_map_reason
    sc = _scenario()
    assert big_map_reason(sc.map.grid_w, sc.map.grid_h) is None
    env = _env(sc, 4)
    ctas = C.c_int32(-1)
    assert env.lib.rlca_env_lidar_ctas_per_sm(env._h, C.byref(ctas)) == 0 and ctas.value >= 1
    rnd = _env_random(4)
    assert env.lib.rlca_env_lidar_ctas_per_sm(rnd._h, C.byref(ctas)) == 0 and ctas.value == 0


def _env_random(W):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    return StageWorld(512, scenario=make_scenario('random'), num_worlds=W, auto_reset=0)


def _controllers(env, kind):
    from rl_collision_avoidance_b200.crowd import Crowd
    from rl_collision_avoidance_b200.dwa import DwaController
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    from rl_collision_avoidance_b200.orca import NhOrcaController
    kw = {}
    if kind == 'policy':
        pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
        pol.load_state_dict(torch.load(STAGE2, map_location='cuda'))
    elif kind == 'nh-orca':
        pol = NhOrcaController(env, obstacles=True)
    elif kind == 'dwa':
        pol = DwaController(env)
    else:                                     # the policy among a map-aware crowd of 2 per world
        pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
        pol.load_state_dict(torch.load(STAGE2, map_location='cuda'))
        kw['crowd'] = Crowd(env, non_cooperative_mask(env.num_env, env.num_worlds, 2), obstacles=True)
    return pol, kw


@pytest.mark.parametrize('kind', ['policy', 'nh-orca', 'dwa', 'crowd'])
def test_evaluate_is_deterministic_and_shard_invariant(built, kind):
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.scenarios import random_max_ticks
    sc = _scenario(8, 64, 0)
    ticks = random_max_ticks(sc.layout.side)

    def run(W, wo):
        env = _env(sc, W, seed=5, world_offset=wo)
        pol, kw = _controllers(env, kind)
        return evaluate(env, pol, 1, ticks, check_every=50, safety=0.1, progress={}, **kw)

    a, b = run(16, 0), run(16, 0)
    assert np.array_equal(a['partials'], b['partials']) and a['ticks'] == b['ticks']
    m = a['metrics']
    assert m['episodes'] > 0 and (kind == 'crowd' or m['episodes'] + m['unfinished'] == 128)
    parts = [run(10, 0), run(6, 10)]
    assert np.array_equal(np.concatenate([p['partials'] for p in parts]), a['partials'])
    # the totals are float64 sums over worlds: the same up to the order of the additions
    assert np.allclose(sum(p['totals'] for p in parts), a['totals'], rtol=1e-12, atol=0)


def test_evaluate_cli_json_is_reproducible(built, tmp_path):
    import evaluate
    outs = []
    for i in range(2):
        path = tmp_path / f'{i}.json'
        evaluate.main(['--scenario', 'arena', '--policy', STAGE2, '--num-worlds', '32', '--arena-robots', '8',
                       '--arena-count', '16', '--arena-seed', '3', '--seed', '2', '--safety', '--timeouts',
                       '--scan-noise', '0.02', '--command-delay', '1', '--json', str(path)])
        outs.append(json.loads(path.read_text()))
    assert outs[0]['partials'] == outs[1]['partials'] and outs[0]['metrics'] == outs[1]['metrics']
    m = outs[0]['metrics']
    assert outs[0]['args']['arena_seed'] == 3 and m['episodes'] > 0 and m['episodes'] + m['unfinished'] == 256
    held = evaluate.main(['--scenario', 'arena', '--baseline', 'nh-orca', '--orca-map', '--num-worlds', '8',
                          '--arena-seed', '9', '--non-cooperative', '2'])
    assert held['metrics']['episodes'] > 0


def _ppo(tmp_path, argv, tag):
    env = dict(os.environ, PYTHONPATH=ROOT)
    d = tmp_path / tag
    d.mkdir()
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'ppo_stage2.py')] + argv +
                       ['--policy-path', str(d / 'policy')], cwd=d, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout, d


def _episode_log(d):
    """The per-episode lines of a run's log/<host>/output.log, without their time stamps."""
    (host,) = os.listdir(d / 'log')
    lines = (d / 'log' / host / 'output.log').read_text().splitlines()
    return [l.split(' - INFO - ', 1)[1] for l in lines if ' - INFO - Env ' in l]


def test_ppo_stage2_arena_end_to_end(built, tmp_path):
    out, d = _ppo(tmp_path, ['--scenario', 'arena', '--arena-robots', '8', '--arena-count', '16', '--arena-timeout',
                             '60', '--num-worlds', '16', '--updates', '2', '--seed', '3'], 'cli')
    assert 'update 2:' in out
    assert any('Crashed' in l or 'Reach Goal' in l or 'Time out' in l for l in _episode_log(d))


def _train(seed, updates=2):
    """trainer.run on 16 arena worlds (pick 1, 40-tick time-out) from stage2.pth with a seeded shuffle."""
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.trainer import run
    env = _started(_scenario(8, 16, 1, timeout=40), 16, seed=seed)
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(128, env.N))
    policy.load_state_dict(torch.load(STAGE2, map_location='cuda'))
    before = policy.flat.clone()
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=64, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=128, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=8, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    stats = run(env=env, policy=policy, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp,
                stage=2, max_updates=updates, generator=torch.Generator(device='cuda').manual_seed(seed))
    return env, policy, before, stats


def test_training_on_arenas_is_deterministic(built):
    a, b = _train(4), _train(4)
    assert len(a[3]) == 2 and all(np.isfinite(s['losses']).all() for s in a[3])
    assert float((a[1].flat - a[2]).abs().max()) > 0
    assert _tsame(a[1].flat, b[1].flat)
    for k in ('pose', 'goal', 'acc', 'meta'):
        assert _tsame(a[0].state[k], b[0].state[k]), k
    assert int(a[0].state['meta'][:, 1].max()) >= 2                     # worlds were re-laid


def test_ppo_stage2_mix_with_arena_trains(built, tmp_path):
    out, _ = _ppo(tmp_path, ['--mix', 'stage2:2,arena:16', '--arena-count', '8', '--arena-timeout', '60',
                             '--updates', '2'], 'mix')
    assert 'update 2:' in out and '  arena: 16 worlds x 8 robots' in out, out[-2000:]
