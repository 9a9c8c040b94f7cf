"""The dynamic-window baseline on the device (DESIGN.md §9u): rlca_dwa_action against its host twin bit for bit on env
states of stage 1, stage 2, the circle and random layouts, at several grid sizes with and without window limits, and
on stacks perturbed by noise and latency; inside evaluate() (what the controller read and what reached the tick, under
scan noise, scan delay and localization error, on the circle and among a crowd); and evaluate.py --baseline dwa."""
import json

import numpy as np
import pytest
import torch

from helpers import random_actions

pytestmark = pytest.mark.gpu


def _env(scenario, worlds, seed, R=None):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    if scenario == 'random':
        sc = make_scenario('random', robots_per_world=R, side=10.0)
    else:
        sc = scenario
    return StageWorld(512, scenario=sc, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same(dwa, stack, gs):
    from rl_collision_avoidance_b200.dwa import dwa_host
    act = dwa(stack, gs)
    torch.cuda.synchronize()
    want, status = dwa_host(dwa.env.cfg, stack.cpu().numpy(), gs.cpu().numpy(), dwa.params)
    assert np.array_equal(_bits(act.cpu().numpy()), _bits(want))
    assert np.array_equal(dwa.status().cpu().numpy(), status)
    return status


PARAMS = [dict(), dict(v_samples=1, w_samples=1), dict(v_samples=32, w_samples=32), dict(v_samples=5, w_samples=3),
          dict(accel=1.0, angular_accel=2.0), dict(v_samples=7, w_samples=40, accel=0.5, angular_accel=0.5,
                                                    radius=0.5, horizon=3.0, brake=0.5)]


@pytest.mark.parametrize('scenario,worlds,R', [('stage1', 171, None), ('stage2', 8, None), ('circle', 4, None),
                                               ('random', 12, 16)])
def test_kernel_matches_host_twin(built, scenario, worlds, R):
    """After 25 random-action ticks through the env's FIFO, every grid and window of PARAMS, bit for bit; both
    statuses occur over the sweep."""
    from rl_collision_avoidance_b200.dwa import DwaController, DwaParams
    env = _env(scenario, worlds, seed=17, R=R)
    env.reset_pose()
    if env.sc.layout is not None:
        env.random_layout()
    rng = np.random.default_rng(17)
    stacks = [env.obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, 512, device=env.device)]
    for t in range(25):
        a = torch.from_numpy(random_actions(rng, env.N)).cuda()
        env.control_vel(a, stack_in=stacks[t & 1], stack_out=stacks[1 - (t & 1)])
    stack = stacks[1]
    seen = set()
    for kw in PARAMS:
        st = _same(DwaController(env, DwaParams(**kw)), stack, env.gs)
        seen |= set(np.unique(st).tolist())
    # a stack whose newest frame holds returns within the radius and a believed speed outside the action box
    s2 = stack.clone()
    s2[::5, 2, 200:300] = -0.49
    g2 = env.gs.clone()
    g2[::3, 2:4] = torch.tensor([1.7, -2.5], device=env.device)
    st = _same(DwaController(env, DwaParams(accel=1.0, angular_accel=1.0)), s2, g2)
    seen |= set(np.unique(st).tolist())
    assert seen == {0, 1}, seen


def test_kernel_matches_host_twin_on_perturbed_stacks(built):
    from rl_collision_avoidance_b200.dwa import DwaController, DwaParams
    from rl_collision_avoidance_b200.latency import Latency, LatencyParams
    from rl_collision_avoidance_b200.noise import Noise, NoiseParams
    env = _env('stage2', 6, seed=4)
    env.reset_pose()
    noise = Noise(env, NoiseParams(range_sigma=0.1, dropout=0.2, seed=5))
    lat = Latency(env, LatencyParams(scan_delay=(1, 3), seed=6))
    rng = np.random.default_rng(4)
    stacks = [env.obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, 512, device=env.device)]
    lat.scan(stacks[0])
    noise.scan(stacks[0])
    dwa = DwaController(env, DwaParams())
    for t in range(12):
        k = t & 1
        if t % 4 == 3:
            _same(dwa, stacks[k], env.gs)
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda(), stack_in=stacks[k],
                        stack_out=stacks[1 - k])
        lat.scan(stacks[1 - k], env.flags)
        noise.scan(stacks[1 - k], env.flags)


def _recorder():
    from rl_collision_avoidance_b200.dwa import DwaController

    class Recorded(DwaController):
        """Logs the stack, gs and action of every call."""

        def __init__(self, *args, **kw):
            super().__init__(*args, **kw)
            self.reads = []

        def __call__(self, stack, gs):
            act = super().__call__(stack, gs)
            self.reads.append((stack.cpu().numpy(), gs.cpu().numpy(), act.cpu().numpy()))
            return act
    return Recorded


@pytest.mark.parametrize('case', ['noise', 'latency', 'localization', 'circle', 'crowd'])
def test_evaluate_drives_with_what_the_controller_read(built, case):
    """Every tick: the controller's action equals the twin's on the stack and gs it was given, and the command the
    tick receives is that action (sensing perturbations do not touch the command), with v = 0 on finished circle
    robots, and the crowd's own rows among a crowd."""
    from rl_collision_avoidance_b200.crowd import Crowd, crowd_host
    from rl_collision_avoidance_b200.dwa import DwaParams, dwa_host
    from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask
    from rl_collision_avoidance_b200.latency import Latency, LatencyParams
    from rl_collision_avoidance_b200.localization import Localization, LocalizationParams
    from rl_collision_avoidance_b200.noise import Noise, NoiseParams
    env = _env('circle' if case == 'circle' else 'stage2', 2, seed=9)
    kw = {}
    if case == 'noise':
        kw['noise'] = Noise(env, NoiseParams(range_sigma=0.05, dropout=0.1, seed=1))
    elif case == 'latency':
        kw['latency'] = Latency(env, LatencyParams(scan_delay=(2, 2), seed=2))
    elif case == 'localization':
        kw['localization'] = Localization(env, LocalizationParams(pose_sigma=(0.1, 0.3), heading_sigma=(0.05, 0.05),
                                                                  speed_sigma=(0.05, 0.1), seed=3))
    mask = None
    if case == 'crowd':
        mask = non_cooperative_mask(env.cfg.robots_per_world, 2, 5)
        kw['crowd'] = Crowd(env, mask, obstacles=True)
    dwa = _recorder()(env, DwaParams())
    sent = []
    step = env.control_vel

    def control_vel(action, **kw):
        st = env.state
        sent.append((st['pose'].cpu().numpy(), st['goal'].cpu().numpy(), st['meta'].cpu().numpy(),
                     action.cpu().numpy()))
        step(action, **kw)
    env.control_vel = control_vel
    out = evaluate(env, dwa, 1, max_ticks=120, check_every=10, progress={}, **kw)
    env.control_vel = step
    reads = dwa.reads
    assert len(reads) == len(sent) == out['ticks'] > 0
    for t in range(0, out['ticks'], 3):
        stack, gs, act = reads[t]
        want, _ = dwa_host(env.cfg, stack, gs, dwa.params)
        assert np.array_equal(_bits(act), _bits(want)), t
        pose, goal, meta, cmd = sent[t]
        if case == 'crowd':
            exp = crowd_host(env.cfg, pose, goal, meta, mask, act, kw['crowd'].params, obstacles=kw['crowd'].obstacles)
            assert np.array_equal(_bits(cmd), _bits(exp)), t
            assert np.array_equal(_bits(cmd[mask == 0]), _bits(act[mask == 0]))
        elif case == 'circle':
            assert np.array_equal(_bits(cmd[:, 1]), _bits(act[:, 1]))
            assert ((cmd[:, 0] == act[:, 0]) | (cmd[:, 0] == 0)).all()
        else:
            assert np.array_equal(_bits(cmd), _bits(act)), t
    if case == 'localization':
        assert any(not np.array_equal(r[1], s[1]) for r, s in zip(reads[1:], reads[:-1]))
    assert 0.0 <= out['dwa']['fallback_share'] <= 1.0 and out['dwa']['v_samples'] == 11


def test_evaluate_refuses_hybrid_and_foreign_env(built):
    from rl_collision_avoidance_b200.dwa import DwaController
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import Hybrid
    env, other = _env('stage2', 1, seed=0), _env('stage2', 1, seed=1)
    with pytest.raises(ValueError, match='hybrid switches a policy'):
        evaluate(env, DwaController(env), 1, 10, hybrid=Hybrid(env))
    with pytest.raises(ValueError, match='another env'):
        evaluate(env, DwaController(other), 1, 10)


def test_evaluate_cli_json_is_reproducible(built, tmp_path, capsys):
    import evaluate
    parts = []
    for i in range(2):
        path = tmp_path / ('dwa%d.json' % i)
        evaluate.main(['--scenario', 'stage2', '--baseline', 'dwa', '--num-worlds', '2', '--episodes', '1',
                       '--max-ticks', '150', '--scan-noise', '0.05', '--beam-dropout', '0.1', '--scan-delay', '2',
                       '--pose-error', '0.1,0.3', '--timeouts', '--seed', '7', '--json', str(path)])
        d = json.loads(path.read_text())
        assert d['controller'] == 'dwa' and d['robots'] == 88
        assert d['dwa']['v_samples'] == 11 and 0.0 <= d['dwa']['fallback_share'] <= 1.0
        assert 'noise' in d and 'latency' in d and 'localization' in d
        assert not any(k.startswith('orca') and d['args'][k] not in (None, False) for k in ('orca_map', 'orca_gain'))
        parts.append(d['partials'])
    out = capsys.readouterr().out
    assert 'dwa  stage2  robots 88' in out and 'dwa  fallback share' in out
    assert parts[0] == parts[1]
