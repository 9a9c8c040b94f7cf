"""The social-force crowd on the device (DESIGN.md §9t): rlca_crowd_action against its host twin at the bench shape,
on stage 2, the circle, stage 1 at R = 1 and random layouts at R = 44 and 64, with every kind of mask, map-blind and with the map;
inside evaluate() (the action the tick receives, the split reduction, an all-zero mask against the recorded
partials); the head-on pair; and rollouts and PPO updates with a crowd and with non-cooperative robots, whose masked
rows no update sees."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import random_actions

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _policy(name, n):
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, name), map_location='cpu'))
    return pol


def _env(scenario, worlds, seed, R=None):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    if scenario == 'random':
        sc = make_scenario('random', robots_per_world=R, side=16.0 if R > 16 else 10.0)
    else:
        sc = make_scenario(scenario, robots_per_world=R) if R is not None else scenario
    return StageWorld(512, scenario=sc, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])


def _host_state(env):
    st = env.state
    return st['pose'].cpu().numpy(), st['goal'].cpu().numpy(), st['meta'].cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize('scenario,worlds,R', [('stage1', 171, None), ('stage2', 8, None), ('circle', 4, None),
                                               ('stage1', 300, 1), ('random', 12, 44), ('random', 9, 64)])
def test_kernel_matches_host_twin(built, scenario, worlds, R):
    """After 25 random-action ticks: no, all, evenly spaced and random masks, map-blind and with the map, seeing and
    ignoring the robots; every row bit for bit, unmasked rows keep a NaN-laced sentinel."""
    from rl_collision_avoidance_b200.crowd import Crowd, CrowdParams, crowd_host
    from rl_collision_avoidance_b200.evaluation import non_cooperative_mask
    from rl_collision_avoidance_b200.orca import ObstacleSet
    env = _env(scenario, worlds, seed=31, R=R)
    env.reset_pose()
    if env.sc.layout is not None:
        env.random_layout()
    rng = np.random.default_rng(31)
    for _ in range(25):
        env.control_vel(torch.from_numpy(random_actions(rng, env.N)).cuda())
    pose, goal, meta = _host_state(env)
    Rw, W = env.cfg.robots_per_world, env.num_worlds
    masks = {'none': np.zeros(env.N, np.uint8), 'all': np.ones(env.N, np.uint8),
             'spaced': non_cooperative_mask(Rw, W, min(5, Rw)),
             'random': (rng.random(env.N) < 0.4).astype(np.uint8) * rng.integers(1, 256, env.N).astype(np.uint8)}
    with torch.cuda.device(env.device):
        obs = ObstacleSet(env.cfg, env.sc.map.cells, 1.0)
    settings = [(CrowdParams(), None), (CrowdParams(), obs), (CrowdParams(see_robots=False, speed=0.6), obs),
                (CrowdParams(side_bias=0.0, anisotropy=1.0, heading_gain=0.8), None)]
    for name, mask in masks.items():
        for k, (p, o) in enumerate(settings):
            act0 = rng.uniform(-3, 3, (env.N, 2)).astype(np.float32)
            act0[::11, 1] = np.nan
            act = torch.from_numpy(act0).cuda()
            Crowd(env, mask, p, obstacles=o).apply(act)
            got = act.cpu().numpy()
            want = crowd_host(env.cfg, pose, goal, meta, mask, act0, p, obstacles=o)
            assert np.array_equal(_bits(got), _bits(want)), (name, k)
            keep = mask == 0
            assert np.array_equal(_bits(got[keep]), _bits(act0[keep])), (name, k)
            if mask.any():
                assert not np.array_equal(_bits(got[~keep]), _bits(act0[~keep])), (name, k)


def test_override_reaches_the_tick_and_split_matches_host(built):
    """Inside evaluate() on stage 2 with the map: the action every tick receives on the crowd's rows is the twin's
    from the state before the tick, the other rows are the policy's; partials_split equals
    rlca_eval_reduce_split_host and 'by_role' holds its rows."""
    from rl_collision_avoidance_b200.crowd import Crowd, crowd_host
    from rl_collision_avoidance_b200.evaluation import evaluate, metrics, non_cooperative_mask, reduce_split_host, \
        totals
    env = _env('stage2', 3, seed=2)
    mask = non_cooperative_mask(env.cfg.robots_per_world, 3, 5)
    crowd = Crowd(env, mask, obstacles=True)
    log = []
    step = env.control_vel

    def control_vel(action, **kw):
        log.append((*_host_state(env), action.cpu().numpy()))
        step(action, **kw)

    env.control_vel = control_vel
    out = evaluate(env, _policy('stage2.pth', env.N), 2, max_ticks=402, crowd=crowd, safety=0.1, progress={})
    env.control_vel = step
    assert len(log) == out['ticks']
    for pose, goal, meta, sent in log[::7]:
        want = crowd_host(env.cfg, pose, goal, meta, mask, sent, crowd.params, obstacles=crowd.obstacles)
        assert np.array_equal(_bits(sent), _bits(want))
    tr = out['tracker']
    host = reduce_split_host(env.cfg, tr.records.cpu().numpy(), tr.count.cpu().numpy(), tr.open.cpu().numpy(), mask)
    split = out['partials_split']
    assert np.array_equal(host.view(np.uint64), split.view(np.uint64))
    by = out['by_role']
    assert set(by) == {'cooperative', 'crowd'} and set(out['safety_by_role']) == {'cooperative', 'crowd'}
    assert set(out['progress_by_role']) == {'cooperative', 'crowd'}
    assert by['crowd']['episodes'] > 0 and by['cooperative']['episodes'] > 0
    for role, row in (('cooperative', 0), ('crowd', 1)):
        want = metrics(totals(split[:, row]))
        assert all(by[role][k] == want[k] for k in ('episodes', 'reached', 'crashed', 'timed_out', 'unfinished'))


def test_evaluate_refuses_both_kinds(built):
    from rl_collision_avoidance_b200.crowd import Crowd
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import NonCooperative
    env = _env('stage2', 1, seed=0)
    m = np.ones(env.N, np.uint8)
    with pytest.raises(ValueError):
        evaluate(env, _policy('stage2.pth', env.N), 1, 10, non_cooperative=NonCooperative(env, m), crowd=Crowd(env, m))
    other = _env('stage2', 1, seed=0)
    with pytest.raises(ValueError):
        evaluate(env, _policy('stage2.pth', env.N), 1, 10, crowd=Crowd(other, m))


@pytest.mark.parametrize('name', ['stage1_policy', 'circle_orca'])
def test_all_zero_mask_changes_nothing(built, name):
    """An all-zero mask, map-aware: the partials recorded before the feature existed, bit for bit."""
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_golden_eval
    from rl_collision_avoidance_b200.crowd import Crowd
    from rl_collision_avoidance_b200.evaluation import evaluate
    from rl_collision_avoidance_b200.orca import NhOrcaController, OrcaController
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_partials.npz'))
    scenario, worlds, seed, who, episodes, max_ticks, check_every = make_golden_eval.RUNS[name]
    env = _env(scenario, worlds, seed)
    policy = OrcaController(env) if who == 'orca' else NhOrcaController(env, obstacles=True) if who == 'nh-orca' \
        else _policy(who, env.N)
    out = evaluate(env, policy, episodes, max_ticks, check_every=check_every,
                   crowd=Crowd(env, np.zeros(env.N, np.uint8), obstacles=True))
    assert out['ticks'] == int(g['ticks_' + name])
    assert np.array_equal(out['partials'].view(np.uint64), g['partials_' + name].view(np.uint64))
    assert not out['partials_split'][:, 1].any()


def test_head_on_crowd_pair_does_not_crash(built):
    """§9h's K = 2, r = 4 m circle, where two straight drivers crash head-on: two crowd agents with the defaults reach
    their goals."""
    import evaluate
    out = evaluate.main(['--scenario', 'circle', '--circle-robots', '2', '--circle-radius', '4', '--baseline', 'orca',
                         '--crowd', '2', '--max-ticks', '300', '--check-every', '10'])
    by = out['by_role']['crowd']
    assert by['crashed'] == 0 and by['reached'] == 2, by


def test_evaluate_cli_json(built, tmp_path, capsys):
    import json

    import evaluate
    path = tmp_path / 'crowd.json'
    evaluate.main(['--scenario', 'stage2', '--policy', os.path.join(CKPT, 'stage2.pth'), '--num-worlds', '2',
                   '--episodes', '1', '--max-ticks', '150', '--crowd', '5', '--crowd-map', '--crowd-ignores-robots',
                   '--json', str(path)])
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 3 and lines[-1].startswith('crowd  stage2  robots 10'), lines
    d = json.loads(path.read_text())
    assert d['crowd']['map'] and not d['crowd']['see_robots'] and d['crowd']['agents'] == 10
    assert set(d['by_role']) == {'cooperative', 'crowd'}


# ---------------------------------------------------------------------------------------------- training
def _train(envs, stage, updates, monkeypatch, seed=0, **kw):
    """trainer.run with diagnostics; checks that every epoch saw all rows but the filtered ones and that the filter is
    the reference's united with every row of a masked column.  Returns the stats."""
    from rl_collision_avoidance_b200 import trainer
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.model.utils import get_filter_index
    N = sum(e.N for e in envs)
    H, bs = 32, 256
    filters = []
    real_filter, real_rows = trainer.masked_filter_index, trainer.masked_rows

    def masked_filter_index(dones, col):
        f = real_filter(dones, col)
        want = set(int(i) for i in get_filter_index(dones)) | {t * N + i for t in range(H) for i in np.flatnonzero(col)}
        assert f == sorted(want)
        filters.append(len(f))
        return f

    def masked_rows(h, col):
        f = real_rows(h, col)
        assert len(f) == h * int(col.sum()) and len(set(f)) == len(f)
        filters.append(len(f))
        return f

    if stage == 1:
        monkeypatch.setattr(trainer, 'masked_rows', masked_rows)
    else:                                   # its own call of masked_rows stays the real one
        monkeypatch.setattr(trainer, 'masked_filter_index', masked_filter_index)
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(bs, N))
    policy.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth' if stage == 2 else 'stage1_2.pth'),
                                      map_location='cuda'))
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=H, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=bs, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=envs[0].num_env, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    gen = torch.Generator(device='cuda').manual_seed(seed)
    stats = trainer.run(env=envs if len(envs) > 1 else envs[0], policy=policy, policy_path=None,
                        action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp, stage=stage, max_updates=updates,
                        generator=gen, diagnostics=True, **kw)
    assert len(stats) == updates and len(filters) == updates
    for s, nf in zip(stats, filters):
        assert np.isfinite(s['losses']).all()
        kept = H * N - nf
        want = kept if stage == 1 else kept // bs * bs
        assert [e['rows'] for e in s['diagnostics']['per_epoch']] == [want] * 2, (nf, want)
        assert set(s['by_role']) == {'cooperative', 'crowd' if 'crowd' in kw else 'non_cooperative'}
        assert sum(r['episodes'] for r in s['by_role'].values()) == s['episodes']
    assert torch.isfinite(policy.flat).all()
    monkeypatch.undo()
    return stats


def _same_stats(a, b):
    keys = ('episodes', 'mean_ep_reward', 'success_rate', 'losses', 'by_role', 'by_scenario')
    return len(a) == len(b) and all(repr(x[k]) == repr(y[k]) for x, y in zip(a, b) for k in keys)


@pytest.mark.parametrize('kind', ['crowd', 'non_cooperative'])
def test_training_with_masked_agents(built, monkeypatch, kind):
    """Stage 1 (filter_index of the masked rows), random layouts and a mix (stage 2's filter united with them): finite
    losses, every epoch sees exactly the unfiltered rows, and two seeded runs give identical stats."""
    from rl_collision_avoidance_b200.crowd import CrowdParams
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from test_mix_gpu import _envs
    kw = {'crowd': (2, CrowdParams(), True)} if kind == 'crowd' else {'non_cooperative': (2, 0.8)}
    s1 = lambda: [StageWorld(512, scenario='stage1', num_worlds=4, seed=1, auto_reset=1)]
    a = _train(s1(), 1, 2, monkeypatch, **kw)
    b = _train(s1(), 1, 2, monkeypatch, **kw)
    assert _same_stats(a, b)
    _train(_envs(seed=2, names=('random',)), 2, 2, monkeypatch, **kw)
    c = _train(_envs(seed=2), 2, 2, monkeypatch, **kw)
    d = _train(_envs(seed=2), 2, 2, monkeypatch, **kw)
    assert _same_stats(c, d)


def test_masked_rows_keep_the_sampled_action(built):
    """In a rollout the masked columns' ro.actions hold the policy's samples while the tick executes the crowd's action:
    the action the env receives on those rows equals the twin's."""
    from rl_collision_avoidance_b200.crowd import CrowdParams, crowd_host
    from rl_collision_avoidance_b200.model.ppo import generate_action
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from rl_collision_avoidance_b200.trainer import Rollout, compose, masked_agents
    env = StageWorld(512, scenario='stage1', num_worlds=4, seed=3, auto_reset=1)
    pol = _policy('stage1_2.pth', env.N)
    ro = Rollout(8, env.N, 512, 'cuda')
    comps = compose([env], ro)
    col = masked_agents(comps, crowd=(3, CrowdParams(), False))
    comps[0].start()
    step = env.control_vel
    sent = []

    def control_vel(action, **kw):
        sent.append((*_host_state(env), action.cpu().numpy()))
        step(action, **kw)

    env.control_vel = control_vel
    for t in range(8):
        generate_action(env=env, state_list=(ro.stacks[t], ro.gs[t]), policy=pol, action_bound=[[0, -1], [1, 1]],
                        out={'value': ro.values[t], 'action': ro.actions[t], 'logprob': ro.logprobs[t],
                             'scaled': ro.scaled})
        scaled = ro.scaled.cpu().numpy()
        comps[0].tick(t)
        pose, goal, meta, act = sent[-1]
        want = crowd_host(env.cfg, pose, goal, meta, col.astype(np.uint8), scaled)
        assert np.array_equal(_bits(act), _bits(want)), t
        assert not np.array_equal(_bits(act[col]), _bits(scaled[col]))
    env.control_vel = step
    assert torch.isfinite(ro.actions).all()
