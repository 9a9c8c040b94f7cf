"""Random layouts on the device (DESIGN.md §9i): rlca_layout_random against its host twin, the env after a layout
against the CPU oracle, the first tick of a tightly packed layout, and evaluate() / evaluate.py on random scenarios."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from helpers import assert_outputs_equal, assert_state_equal, random_actions

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _scenario(K, S=10.0, D=1.0, L=None):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    return make_scenario('random', robots_per_world=K, side=S, separation=D, min_travel=L)


def _env(sc, W, seed=0, world_offset=0, max_reject=4096):
    """A random-scenario env right after the reset evaluate() runs, before the layout."""
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=sc, num_worlds=W, seed=seed, auto_reset=0, world_offset=world_offset,
                     max_reject=max_reject)
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    return env


def _host_rows(env):
    torch.cuda.synchronize()
    return tuple(env.state[k].cpu().numpy() for k in ('pose', 'goal', 'acc'))


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _multi_round(sc, cfg):
    """True when some robot of cfg's worlds needs more than 32 tries: the host twin fails with a 32-try budget."""
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.scenarios import random_layout_host
    c = _lib.EnvConfig.from_buffer_copy(cfg)
    c.max_reject = 32
    z = np.zeros((sc.robots_per_world * c.num_worlds, 4), np.float32)
    return bool(random_layout_host(c, sc.layout, z, z, z)[3].any())


@pytest.mark.parametrize('K,S,W,seed', [(4, 10.0, 4096, 0), (8, 10.0, 4096, 1), (64, 20.0, 1024, 2),
                                        (64, 20.0, 37, 3)])
def test_device_equals_host(built, K, S, W, seed):
    from rl_collision_avoidance_b200.scenarios import random_layout_host
    sc = _scenario(K, S)
    env = _env(sc, W, seed)
    before = _host_rows(env)
    want = random_layout_host(env.cfg, sc.layout, *before)
    assert not want[3].any()
    env.random_layout()
    for name, got, ref in zip(('pose', 'goal', 'acc'), _host_rows(env), want[:3]):
        assert _bits_equal(got, ref), name
    meta = env.state['meta'].cpu().numpy()
    assert (meta[:, 1] == 1).all()                              # the episode reset_pose started is kept
    if K == 64 and W == 1024:
        assert _multi_round(sc, env.cfg)


def test_device_failure_status_equals_host(built):
    """A 16-robot layout in an 8 m square with 8 tries: the device's per-world status equals the host twin's, failed
    worlds keep their rows, and random_layout() names the first failed world."""
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.scenarios import random_layout_host
    sc = _scenario(16, 8.0)
    env = _env(sc, 64, seed=0, max_reject=8)
    before = _host_rows(env)
    want = random_layout_host(env.cfg, sc.layout, *before)
    assert want[3].any() and not want[3].all()
    status = torch.full((64,), -1, dtype=torch.int32, device='cuda')
    params = _lib.LayoutParams(sc.layout.side, sc.layout.separation, sc.layout.min_travel)
    st = env._state_struct(env._cur)
    _lib.check(env.lib.rlca_layout_random(C.byref(env.cfg), C.byref(params), C.byref(st),
                                          C.c_void_p(status.data_ptr()), None))
    assert np.array_equal(status.cpu().numpy(), want[3])
    for got, ref in zip(_host_rows(env), want[:3]):
        assert _bits_equal(got, ref)
    env2 = _env(sc, 64, seed=0, max_reject=8)
    w = int(np.flatnonzero(want[3])[0])
    with pytest.raises(ValueError, match=f'world {w}: robot {int(want[3][w]) - 1} not placed in 8 tries'):
        env2.random_layout()


def test_crowded_layout_raises(built):
    env = _env(_scenario(64, 6.0, 1.0, 3.0), 2)
    with pytest.raises(ValueError, match='world 0: robot 29 not placed in 4096 tries; lower the density'):
        env.random_layout()


def test_world_offset_shards_give_one_handles_rows(built):
    sc = _scenario(8)
    one = _env(sc, 200, seed=4)
    one.random_layout()
    rows = _host_rows(one)
    parts = []
    for w0, wc in ((0, 120), (120, 80)):
        e = _env(sc, wc, seed=4, world_offset=w0)
        e.random_layout()
        parts.append(_host_rows(e))
    for i in range(3):
        assert _bits_equal(np.concatenate([p[i] for p in parts]), rows[i])


@pytest.mark.parametrize('K,S,W', [(8, 10.0, 16), (64, 20.0, 4)])
def test_oracle_parity_after_layout(built, K, S, W):
    """The layout copied into the oracle: scan and local goal equal, then 20 random-action ticks with auto_reset 0
    stay bit-exact in state, scan, local goal and flags."""
    from oracle.oracle import OracleWorld, OrcConfig
    from rl_collision_avoidance_b200.scenarios import fill_config
    sc = _scenario(K, S)
    env = _env(sc, W, seed=7)
    env.random_layout()
    ocfg = fill_config(OrcConfig(), sc, num_worlds=W, beams=512, auto_reset=0, seed=7)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    torch.cuda.synchronize()
    for k in ('pose', 'goal', 'acc', 'meta'):
        getattr(orc, k)[...] = env.state[k].cpu().numpy()
    orc.observe()
    assert_outputs_equal(env, orc, 'layout')
    rng = np.random.default_rng(K)
    for t in range(20):
        a = random_actions(rng, orc.N)
        env.control_vel(torch.from_numpy(a).cuda())
        orc.step(a)
        assert_state_equal(env, orc, f'tick {t}')
        assert_outputs_equal(env, orc, f'tick {t}')
        assert np.array_equal(env.flags.cpu().numpy(), orc.flags), f'tick {t}: flags differ'


def test_packed_starts_do_not_collide(built):
    """Separation just above 2 (r_c + sqrt(2) resolution): one zero-action tick over 4096 worlds x 8 robots raises no
    crash flag and no stall."""
    sc0 = _scenario(8)
    hl, hw, res = (float(np.float32(v)) for v in (0.22, 0.19, sc0.map.resolution))
    d = 2.0 * (math.sqrt(hl * hl + hw * hw) + math.sqrt(2.0) * res) + 1e-4
    sc = _scenario(8, 10.0, d)
    env = _env(sc, 4096, seed=8)
    env.random_layout()
    env.control_vel(torch.zeros(env.N, 2, device='cuda'))
    torch.cuda.synchronize()
    assert not env.flags[:, 1].any()
    assert not env.state['meta'][:, 2].any()
    # the layout really is packed: some pair of starts is closer than 2 r_c + 0.05 m
    p = env._st[1 - env._cur]['pose'][:, 0:2].reshape(4096, 8, 2).double()
    dist = torch.cdist(p, p) + torch.eye(8, device='cuda', dtype=torch.float64) * 1e9
    assert float(dist.min()) < d + 0.05


# ---------------------------------------------------------------------------------------------- evaluate()
def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cpu'))
    return pol


def _evaluate(sc, W, seed, who, world_offset=0, nc=None, max_ticks=426):
    from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask
    from rl_collision_avoidance_b200.orca import NhOrcaController, NonCooperative
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=sc, num_worlds=W, seed=seed, auto_reset=0, world_offset=world_offset)
    policy = NhOrcaController(env, obstacles=True) if who == 'nh-orca-map' else _policy(who, env.N)
    ncc = None if nc is None else NonCooperative(env, non_cooperative_mask(sc.robots_per_world, W, nc))
    return evaluate(env, policy, 1, max_ticks, non_cooperative=ncc)


def test_evaluate_random_is_deterministic_and_per_world(built):
    sc = _scenario(8)
    a = _evaluate(sc, 32, 0, 'stage2.pth')
    b = _evaluate(sc, 32, 0, 'stage2.pth')
    assert a['ticks'] == b['ticks']
    assert np.array_equal(a['partials'].view(np.uint64), b['partials'].view(np.uint64))
    p = a['partials']
    assert len(np.unique(p, axis=0)) > 1                       # the worlds are not copies of each other
    m = a['metrics']
    assert m['episodes'] + m['unfinished'] == 32 * 8 and m['episodes'] > 0
    # the recorded straight-line distances are the layouts': at least min_travel
    assert m['reached'] > 0 and a['totals'][12] / m['reached'] >= sc.layout.min_travel - 1e-4


def test_evaluate_random_shards_give_one_handles_totals(built):
    from rl_collision_avoidance_b200.evaluation import totals
    sc = _scenario(8)
    one = _evaluate(sc, 20, 3, 'stage2.pth')
    parts = [_evaluate(sc, wc, 3, 'stage2.pth', world_offset=w0)['partials'] for w0, wc in ((0, 12), (12, 8))]
    assert np.array_equal(np.concatenate(parts).view(np.uint64), one['partials'].view(np.uint64))
    assert np.array_equal(totals(np.concatenate(parts)).view(np.uint64), one['totals'].view(np.uint64))


def test_evaluate_random_with_baseline_and_non_cooperative(built):
    sc = _scenario(8)
    out = _evaluate(sc, 16, 1, 'nh-orca-map')
    assert out['metrics']['episodes'] > 0 and 'by_role' not in out
    out = _evaluate(sc, 16, 1, 'stage2.pth', nc=2)
    assert set(out['by_role']) == {'cooperative', 'non_cooperative'}
    split = out['partials_split']
    assert np.array_equal(split[:, 0, :4] + split[:, 1, :4], out['partials'][:, :4])
    assert out['by_role']['non_cooperative']['episodes'] + out['by_role']['non_cooperative']['unfinished'] == 32


def test_evaluate_cli_random_json_is_deterministic(built, tmp_path, capsys):
    import evaluate
    path = tmp_path / 'random.json'
    argv = ['--scenario', 'random', '--baseline', 'orca', '--orca-map', '--num-worlds', '8', '--random-robots', '6',
            '--random-side', '8', '--non-cooperative', '2', '--json', str(path)]
    out = evaluate.main(argv)
    first = path.read_bytes()
    evaluate.main(argv)
    assert path.read_bytes() == first
    d = json.loads(first)
    assert d['robots'] == 48 and np.asarray(d['partials']).shape == (8, 14)
    assert out['ticks'] <= evaluate.random_max_ticks(8.0)
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 6 and 'non-cooperative  random  robots 16' in lines[-1]
