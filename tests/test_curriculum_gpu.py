"""The arena curriculum on the device (DESIGN.md §9z): the weighted layout, the weighted re-layout with its fused tally
and the update against their host twins bit for bit after every tick of an arena rollout, equal weights against pick
1's kernel, trainer.run's tallies, determinism and checkpointed state, two ranks over gloo, and the command lines."""
import datetime
import json
import os
import queue
import socket
import subprocess
import sys
import traceback

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
STAGE2 = os.path.join(CKPT, 'stage2.pth')


def _scenario(K=8, T=64, pick=1, timeout=None):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    return make_scenario('arena', robots_per_world=K, arenas=T, pick=pick, timeout=timeout)


def _env(sc, W, seed=0, world_offset=0):
    from rl_collision_avoidance_b200.stage_world import StageWorld
    return StageWorld(512, scenario=sc, num_worlds=W, seed=seed, auto_reset=0, world_offset=world_offset)


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _np(t):
    return t.cpu().numpy()


def _steer(gs, noise):
    w = torch.clamp(2.0 * torch.atan2(gs[:, 1], gs[:, 0]) + noise[:, 1], -1.0, 1.0)
    return torch.stack((torch.clamp(1.0 - noise[:, 0].abs(), 0.0, 1.0), w), 1).contiguous()


def _host_state(env, flags):
    torch.cuda.synchronize()
    st = env.state
    return _np(st['pose']), _np(st['goal']), _np(st['acc']), _np(st['meta']), _np(flags)


def _check_update(cur, pending=None):
    """cur.update() against update_host from the state before it, in place."""
    from rl_collision_avoidance_b200.curriculum import update_host
    if pending is not None:
        cur.pending.copy_(torch.from_numpy(pending))
    E, S, P = _np(cur.E), _np(cur.S), _np(cur.pending)
    cur.update()
    want = update_host(E, S, P, cur.params.decay, cur.params.uniform)
    for name, x, y in zip(('E', 'S', 'pending', 'cdf'), (_np(cur.E), _np(cur.S), _np(cur.pending), _np(cur.cdf)),
                          want):
        assert _same(x, y), name
    assert int(cur.folded) == int(P[:cur.T].sum())


def test_kernels_equal_twins_after_every_tick(built):
    """100 ticks on 512 worlds (25-tick time-out) with a crowd-style row mask of 2 robots per world: the weighted
    layout, every re-layout with its tally, and an update every 20 ticks equal their host twins bit for bit."""
    from rl_collision_avoidance_b200.curriculum import ArenaCurriculum, CurriculumParams, layout_host, relayout_host
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    K, W, T, ticks = 8, 512, 64, 100
    sc = _scenario(K, T, timeout=25)
    env = _env(sc, W, seed=7)
    mask = non_cooperative_mask(K, W, 2)
    cur = ArenaCurriculum(env, CurriculumParams(0.8, 0.05), row_mask=mask)
    assert env.curriculum is cur
    rng = np.random.default_rng(1)
    cur.E.copy_(torch.from_numpy((rng.random(T) * 50).astype(np.float32)))
    cur.S.copy_(cur.E * torch.rand(T, device='cuda', generator=torch.Generator('cuda').manual_seed(2)))
    _check_update(cur, rng.integers(0, 30, 2 * T).astype(np.int32))
    w = np.diff(_np(cur.cdf))
    assert w.min() < w.max()
    env.reset_world()
    rows = _host_state(env, env.flags)[:3]
    wa0 = _np(cur.world_arena)
    env.random_layout()
    want = layout_host(env.cfg, sc.layout, _np(cur.cdf), wa0, *rows)
    got = _host_state(env, env.flags)[:3] + (np.zeros(W, np.int32), _np(cur.world_arena))
    for name, x, y in zip(('pose', 'goal', 'acc', 'status', 'world_arena'), got, want):
        assert _same(x, y), name
    stacks = torch.empty(2, env.N, 3, 512, device='cuda')
    stacks[0] = env.obs[:, None, :]
    gs = env.gs.clone()
    flags = torch.zeros(env.N, 4, dtype=torch.uint8, device='cuda')
    gen = torch.Generator(device='cuda').manual_seed(3)
    mask_t = torch.from_numpy(mask != 0).cuda()
    tallied = 0
    for t in range(ticks):
        env.control_vel(_steer(gs, 0.5 * torch.randn(env.N, 2, device='cuda', generator=gen)), live=env.live,
                        stack_in=stacks[0], stack_out=stacks[1], out={'flags': flags, 'gs': gs})
        before = _host_state(env, flags)
        wa, pend = _np(cur.world_arena), _np(cur.pending)
        env.relayout_finished(stacks[1], out={'flags': flags, 'gs': gs})
        want = relayout_host(env.cfg, sc.layout, _np(cur.cdf), wa, pend, mask, *before)
        got = _host_state(env, flags) + (_np(env.live), _np(env._relayout_status), _np(cur.world_arena),
                                         _np(cur.pending))
        for name, x, y in zip(('pose', 'goal', 'acc', 'meta', 'flags', 'live', 'status', 'world_arena', 'pending'),
                              got, want):
            assert _same(x, y), f'tick {t}: {name} differs'
        ended = (flags[:, 0] != 0) & (flags[:, 2] != 0) & ~mask_t
        tallied += int(ended.sum())
        stacks[0].copy_(stacks[1])
        if t % 20 == 19:
            _check_update(cur)
    assert tallied > 0 and int(_np(cur.E).sum()) > 0


def test_equal_weights_reproduce_pick_1(built):
    """uniform = 1 keeps every weight 2^20 through its updates: the curriculum env lays out and re-lays exactly as pick
    1's kernel, state, flags, live and status after every tick."""
    from rl_collision_avoidance_b200.curriculum import ArenaCurriculum, CurriculumParams
    K, W, T = 8, 256, 16
    sc = _scenario(K, T, timeout=20)
    envs = [_env(sc, W, seed=5, world_offset=3) for _ in range(2)]
    cur = ArenaCurriculum(envs[1], CurriculumParams(0.5, 1.0))
    bufs = []
    for e in envs:
        e.reset_world()
        e.random_layout()
        bufs.append((torch.empty(2, e.N, 3, 512, device='cuda'), e.gs.clone(),
                     torch.zeros(e.N, 4, dtype=torch.uint8, device='cuda')))
        bufs[-1][0][0] = e.obs[:, None, :]
    gen = torch.Generator(device='cuda').manual_seed(0)
    for t in range(80):
        noise = 0.5 * torch.randn(envs[0].N, 2, device='cuda', generator=gen)
        for e, (st, gs, fl) in zip(envs, bufs):
            e.control_vel(_steer(gs, noise), live=e.live, stack_in=st[0], stack_out=st[1], out={'flags': fl, 'gs': gs})
            e.relayout_finished(st[1], out={'flags': fl, 'gs': gs})
            st[0].copy_(st[1])
        if t % 10 == 9:
            cur.update()
        for k in ('pose', 'goal', 'acc', 'meta'):
            assert torch.equal(envs[0].state[k], envs[1].state[k]), f'tick {t}: {k}'
        assert torch.equal(bufs[0][2], bufs[1][2]) and torch.equal(envs[0].live, envs[1].live), t
        assert torch.equal(envs[0]._relayout_status, envs[1]._relayout_status), t
        assert torch.equal(bufs[0][1], bufs[1][1]), t
    assert int(envs[0].state['meta'][:, 1].max()) >= 2
    assert (np.diff(_np(cur.cdf)) == 1 << 20).all() and int(cur.folded) >= 0


HP = dict(HORIZON=64, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=128, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1, NUM_ENV=8,
          OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)


def _train(seed, updates=3, policy_path=None, save_every=20, state=None, non_cooperative=None):
    from rl_collision_avoidance_b200.curriculum import CurriculumParams
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.trainer import run
    env = _env(_scenario(8, 16, timeout=40), 16, seed=seed)
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(128, env.N))
    policy.load_state_dict(torch.load(STAGE2, map_location='cuda'))
    opt = Adam(policy.parameters(), lr=5e-5)
    stats = run(env=env, policy=policy, policy_path=policy_path, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=HP,
                stage=2, max_updates=updates, generator=torch.Generator(device='cuda').manual_seed(seed),
                save_every=save_every, curriculum=CurriculumParams(0.7, 0.1), curriculum_state=state,
                non_cooperative=non_cooperative)
    return env, policy, opt, stats


def test_tallies_equal_the_trainers_cooperative_episodes(built):
    env, _, _, stats = _train(2, updates=3, non_cooperative=(2, None))
    for s in stats:
        assert s['curriculum']['episodes'] == s['by_role']['cooperative']['episodes'] > 0, s['update']
        assert s['curriculum']['arenas'] == 16 and 1.0 <= s['curriculum']['effective_arenas'] <= 16.0


def test_training_is_deterministic(built):
    a, b = _train(4), _train(4)
    strip = lambda st: [{k: v for k, v in s.items() if k not in ('rollout_s', 'update_s', 'agent_steps_per_s')}
                        for s in st]
    assert json.dumps(strip(a[3]), sort_keys=True, default=str) == json.dumps(strip(b[3]), sort_keys=True, default=str)
    assert torch.equal(a[1].flat, b[1].flat)
    assert torch.equal(a[2].exp_avg, b[2].exp_avg) and torch.equal(a[2].exp_avg_sq, b[2].exp_avg_sq)
    sa, sb = a[0].curriculum.state_dict(), b[0].curriculum.state_dict()
    for k in ('E', 'S', 'cdf', 'pending'):
        assert torch.equal(sa[k], sb[k]), k
    assert len(set(np.diff(_np(a[0].curriculum.cdf)).tolist())) > 1          # the weights moved apart


def test_checkpoint_restores_the_curriculum(built, tmp_path):
    """The .trainer checkpoint of update 2 holds the state the run's curriculum held after update 2, bit for bit; a run
    resumed from it restores that state before its first layout, which draws from the saved weights."""
    from rl_collision_avoidance_b200.curriculum import ArenaCurriculum, CurriculumParams, layout_host
    env, _, _, _ = _train(6, updates=2, policy_path=str(tmp_path), save_every=2)
    ck = torch.load(str(tmp_path / 'stage2_2.pth.trainer'))
    live = env.curriculum.state_dict()
    assert ck['update'] == 2
    for k in ('E', 'S', 'cdf', 'pending'):
        assert torch.equal(ck['curriculum'][k], live[k]), k
    assert (ck['curriculum']['num_arenas'], ck['curriculum']['arena_seed']) == (16, 0)
    # the resumed run's first layout
    env2 = _env(_scenario(8, 16, timeout=40), 16, seed=9)
    cur = ArenaCurriculum(env2, CurriculumParams(0.7, 0.1))
    cur.load_state_dict(ck['curriculum'])
    env2.reset_world()
    rows = [_np(env2.state[k]) for k in ('pose', 'goal', 'acc')]
    env2.random_layout()
    want = layout_host(env2.cfg, env2.sc.layout, _np(ck['curriculum']['cdf']), np.zeros(16, np.int32), *rows)
    assert _same(_np(env2.state['pose']), want[0]) and _same(_np(cur.world_arena), want[4])
    # trainer.run takes the state and runs on from it
    _, _, _, stats = _train(9, updates=1, state=ck['curriculum'])
    assert stats[0]['curriculum']['episodes'] > 0


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(seconds=180))
    try:
        from rl_collision_avoidance_b200.curriculum import ArenaCurriculum, CurriculumParams
        W = 64
        env = _env(_scenario(8, 16, timeout=20), W, seed=1, world_offset=rank * W)
        cur = ArenaCurriculum(env, CurriculumParams(0.9, 0.1))
        env.reset_world()
        env.random_layout()
        stack = torch.empty(env.N, 3, 512, device='cuda')
        gs = env.gs.clone()
        flags = torch.zeros(env.N, 4, dtype=torch.uint8, device='cuda')
        gen = torch.Generator(device='cuda').manual_seed(rank)
        res = []
        for u in range(2):
            for _ in range(30):
                env.control_vel(_steer(gs, 0.5 * torch.randn(env.N, 2, device='cuda', generator=gen)), live=env.live,
                                out={'flags': flags, 'gs': gs})
                env.relayout_finished(stack, out={'flags': flags, 'gs': gs})
            before = (_np(cur.E), _np(cur.S), _np(cur.pending))
            cur.update(process_group=True)
            res.append((before, _np(cur.E), _np(cur.S), _np(cur.cdf), int(cur.folded)))
        out.put((rank, res, None))
    except BaseException:
        out.put((rank, None, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_ranks_hold_the_same_weights(built):
    from rl_collision_avoidance_b200.curriculum import update_host
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = {}
        for _ in procs:
            try:
                rank, r, err = q.get(timeout=600)
            except queue.Empty:
                pytest.fail('a worker did not report within 600 s')
            assert err is None, f'rank {rank} failed:\n{err}'
            res[rank] = r
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    for u in range(2):
        (E0, S0, P0), E, S, cdf, folded = res[0][u]
        (E1, S1, P1), *rest = res[1][u]
        assert _same(E0, E1) and _same(S0, S1)
        assert _same(E, rest[0]) and _same(S, rest[1]) and _same(cdf, rest[2]) and folded == rest[3]
        want = update_host(E0, S0, P0 + P1, 0.9, 0.1)
        assert _same(E, want[0]) and _same(S, want[1]) and _same(cdf, want[3])
        assert folded == int((P0 + P1)[:16].sum()) > 0


def _ppo(tmp_path, argv, tag):
    env = dict(os.environ, PYTHONPATH=ROOT)
    d = tmp_path / tag
    d.mkdir()
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'ppo_stage2.py')] + argv +
                       ['--policy-path', str(d / 'policy')], cwd=d, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


def test_ppo_stage2_arena_curriculum_end_to_end(built, tmp_path):
    out = _ppo(tmp_path, ['--scenario', 'arena', '--arena-robots', '8', '--arena-count', '16', '--arena-timeout', '60',
                          '--num-worlds', '16', '--updates', '2', '--seed', '3', '--arena-curriculum',
                          '--curriculum-decay', '0.8'], 'cli')
    assert 'update 2:' in out and 'last update, curriculum: 16 arenas, effective' in out, out[-2000:]


def test_ppo_stage2_mix_with_arena_curriculum(built, tmp_path):
    out = _ppo(tmp_path, ['--mix', 'stage2:2,arena:16', '--arena-count', '8', '--arena-timeout', '60', '--updates', '2',
                          '--arena-curriculum'], 'mix')
    assert 'update 2:' in out and 'last update, curriculum: 8 arenas' in out, out[-2000:]


def test_evaluate_per_arena_json_is_reproducible(built, tmp_path):
    import evaluate
    outs = []
    for i in range(2):
        path = tmp_path / f'{i}.json'
        evaluate.main(['--scenario', 'arena', '--policy', STAGE2, '--num-worlds', '32', '--arena-count', '16',
                       '--arena-seed', '1', '--per-arena', '--timeouts', '--json', str(path)])
        outs.append(json.loads(path.read_text()))
        del outs[-1]['args']['json']
    assert json.dumps(outs[0]) == json.dumps(outs[1])
    res = outs[0]
    rows = res['per_arena']
    assert [r['arena'] for r in rows] == list(range(16)) and all(r['worlds'] == 2 for r in rows)
    assert sum(r['episodes'] for r in rows) == res['metrics']['episodes']
    assert sum(r['unfinished'] for r in rows) == res['metrics']['unfinished']
