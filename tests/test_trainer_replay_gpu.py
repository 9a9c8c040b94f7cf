"""trainer.run replayed on the host: two PPO updates of the unmodified trainer, recorded through wrappers of the names
trainer imports and of the optimizer instance, then every update replayed against independent references.

a. The environment, bit for bit: one CPU oracle per component, driven by the executed commands, with the scan deque of
   tests/trainer_ref.py, the layout and re-layout host twins (random layouts; arenas with the layout's own pick) and
   the noise host twins.  Stacks, goal | speed, rewards, flags and the eplog rows of ended episodes equal the device
   rollout's.  The perturbation chain is restated
   per component and tick: the executed command is the sampled one with the masked rows overridden (the crowd and
   straight-driver host twins on the oracle's state, themselves within their float64 restatements' bounds), then
   latency_ref's command ring, the noise twin and dynamics_ref's limits, the last two links with the flags of the tick
   before; it equals what the env's control_vel received, bit for bit.  The stack is the deque after the re-layout
   refresh, then latency_ref's scan ring and the noise twin; the gs the policy reads is localization_ref's believed gs
   on the oracle's pose and goal after the re-layout.
   With a planner, restated from tests/planner_ref.py alone (PlanReplay), last of all: after the run's start and
   every tick each row whose goal entry changed is re-planned by scipy's Dijkstra, and the device's status equals
   ref.waypoint's on the oracle's pose and goal; the gs the policy reads is the tick's bit for bit where the goal is in
   sight or there is no plan, and the waypoint's local goal within 1e-4 (its speed bit for bit) elsewhere
   (test_waypoint_twin_matches_float64_restatement).  Rows where a tested segment passes within 1e-5 m of a cell
   corner are exempt, at most one in 1000, and carry the device's gs.  With 'geodesic' the device's psi is within
   test_planner_reward's bound of planner_reward_ref.psi, a non-terminal tick's reward within its bound of
   shaped_reward on the tick's reward and the device's psi before and after it, a terminal tick's reward is the tick's
   bit for bit, and an ended episode's return lies within float32 rounding of the float64 sum of the rewards PPO
   trained on (psi_start restarting on flags[:, 3] and at the run's start); its other eplog columns stay bit for bit.
   With 'straight' rewards and eplog stay the tick's., at the weights of the update's start: values against the float64 forward within
   learner_ref.check_forward's bound for the tensor-core mode, means within the bound at _forward64; actions,
   log-probabilities and the clip against sample_ref (test_sample_gpu's bounds); the stored action is the sampled,
   un-noised one; last_v is the float64 value of the replayed state after the horizon.
c. The update: GAE targets and advantages against the float64 recurrence on the rewards checked in a and dones (1 float32
   ulp, test_learner_shapes_gpu.test_gae_vs_float64_recurrence); filter_index exactly; the epochs' permutations drawn
   again from the generator state at entry give the restated minibatch schedule (a ragged last minibatch in stage 1,
   the tail dropped in stage 2) over the rows the restated filter keeps (stage 2: get_filter_index united with every
   row of a masked column; stage 1: those rows alone); then per optimizer step, teacher-forced from the device's parameters at that step, on
   the rows of the replayed minibatch with the restated advantage normalisation (before np.delete): the ppo.log row
   against learner_ref.ref_losses, all 23 gradients against float64 autograd relative to their layer's scale, and the
   Adam step against trainer_ref.adam_step in float64 from the device's gradient (bounds at step_checks and
   adam_bounds).  Every replayed PPO ratio is asserted to be learner_ref.MARGIN away from 1 +- clip.
d. The Env log lines against the replay's own episode bookkeeping, and the stats run returns (episodes, success rate,
   mean episode reward, by_scenario and, with masked agents, by_role) against the eplog rows of ended episodes checked
   in a; with a planner the returns in the lines within a's bound of the float64 sums, and the status shares against
   the replay's statuses over the update's robot-ticks (update 0's with the start's rows).

Real rollouts are not decisive batches (learner_ref): a pre-activation within fp32 rounding of zero can flip its ReLU
mask between the kernels and float64, which moves that tower's gradients by ~1e-3 of their scale.  A tower's tensors are
therefore held to test_learner_gpu's bound for undecided conv masks, 3e-3 of the layer scale, in a minibatch where one
of its conv pre-activations is within learner_ref.MARGIN of its layer's max of zero in float64.  An undecided fc1 / fc2
mask moves its row's whole contribution, so that side's tensors may also differ by twice the float64 gradient of the
rows holding one.  Elsewhere the tight bounds hold.
"""
import collections
import dataclasses
import logging
import math
import os
import time

import numpy as np
import pytest
import torch

import crowd_ref
import dynamics_ref
import latency_ref
import localization_ref
import orca_ref
import planner_ref
import planner_reward_ref as rref
import sample_ref
import trainer_ref as ref
from learner_ref import (CLIP, COEFF, MARGIN, VCOEF, Checks, layer_scale, maxabs, ref_forward, ref_logprob, ref_losses)
from test_crowd import TOL as CROWD_TOL
from test_planner_reward import psi_bound, shaped_bound
from test_sample_gpu import action_bound, lp_bound

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
U = 2.0 ** -24
NOISE = dict(range_sigma=0.05, dropout=0.1, v_gain_sigma=0.2, w_gain_sigma=0.2, seed=2 ** 33 + 5)
LR = 5e-5
B1, B2 = float(np.float32(0.9)), float(np.float32(0.999))      # the betas as the fused Adam kernel receives them
TINY = 2.0 ** -148        # two float32 subnormal steps: the absolute floor of a rounding near zero

LATENCY = dict(scan_delay=(0, 4), command_delay=(1, 3), seed=2 ** 34 + 7)
DYNAMICS = dict(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=2 ** 35 + 9)
LOCALIZATION = dict(pose_sigma=(0.05, 0.2), heading_sigma=(0.02, 0.1), correlation_time=2.0, speed_sigma=(0.05, 0.1),
                    seed=2 ** 36 + 11)
CHAIN_SEED = 1            # the chain's localization seed: with LOCALIZATION's, a PPO ratio falls within MARGIN of 1 + clip
NONCOOP_TOL = 1e-5       # the straight driver's twin against orca_ref's preferred velocity and tracker (test_noncoop)
MIX = [('stage2', 1, 2, 25, {}), ('circle', 2, 2, 100, dict(robots_per_world=8, radius=1.5)),
       ('random', 4, 0, 60, dict(robots_per_world=8, side=6.0))]
# 8 worlds of 8 robots in 16 obstacle arenas of generator seed 2, an arena drawn at every layout (pick 1, as training
# draws them); with a 25-tick time-out every world is re-laid on ticks 25, 51 = H - 1, 77 and 103
ARENA = ('arena', 8, 0, 25, dict(robots_per_world=8, arenas=16, pick=1, arena_seed=2))


def _stage1_pillar():
    """stage 1's map with a 2 m square pillar at its centre: stage 1's room is convex, so only goals behind the
    pillar are out of sight"""
    from rl_collision_avoidance_b200.scenarios import make_scenario
    m = make_scenario('stage1').map
    c = m.cells.copy()
    k = int(round(1.0 / m.resolution))
    c[m.origin_cy - k:m.origin_cy + k, m.origin_cx - k:m.origin_cx + k] = 254
    return dataclasses.replace(m, cells=c, name='stage1 with a pillar')

# (scenario, worlds, auto_reset, timeout, extra make_scenario arguments, a callable one called) per component; the perturbations are the
# keyword arguments of latency.LatencyParams, dynamics.DynamicsParams and localization.LocalizationParams, 'crowd' the
# k of crowd=(k, CrowdParams(), True), 'non_cooperative' the (k, speed) and 'planner' the planner of trainer.run
CASES = {
    # 2 x 24 robots; episodes time out after 20 ticks, so the first ones end on tick 19 and 39 = the horizon's last;
    # H N = 1920 is 7.5 minibatches of 256: a ragged last minibatch
    'stage1': dict(stage=1, comps=[('stage1', 2, 1, 19, {})], H=40, batch=256, ckpt='stage1_2.pth', noise=False),
    # one stage-2 world with a 25-tick time-out: every group re-spawns inside the horizon, early finishers idle
    'stage2': dict(stage=2, comps=[('stage2', 1, 2, 25, {})], H=52, batch=256, ckpt='stage2.pth', noise=False),
    # random layouts under noise: a re-laid row's stack is refreshed before it is perturbed
    'random': dict(stage=2, comps=[('random', 8, 0, 25, dict(robots_per_world=8, side=6.0))], H=52, batch=128,
                   ckpt='stage2.pth', noise=True),
    # stage 2 | circle | random in mix.MIX_SCENARIOS order; the stage-2 groups end together on tick 51 = H - 1, and
    # circle and random robots that finished early idle on update 2's first tick: filter runs cross the boundaries
    'mix': dict(stage=2, comps=MIX, H=52, batch=256, ckpt='stage2.pth', noise=False),
    'noise': dict(stage=1, comps=[('stage1', 2, 1, 19, {})], H=40, batch=256, ckpt='stage1_2.pth', noise=True),
    # stage 1's shape: the episodes ending on tick 39 = H - 1 restart their command rings on update 2's tick 0
    'latency': dict(stage=1, comps=[('stage1', 2, 1, 19, {})], H=40, batch=256, ckpt='stage1_2.pth', noise=False,
                    latency=LATENCY),
    # stage 2's shape: crashed robots' limits restart from 0, groups re-spawn, early finishers idle
    'dynamics': dict(stage=2, comps=[('stage2', 1, 2, 25, {})], H=52, batch=256, ckpt='stage2.pth', noise=False,
                     dynamics=DYNAMICS),
    # random layouts: a re-laid robot's believed gs is drawn from its new layout with fresh sigmas
    'localization': dict(stage=2, comps=[('random', 8, 0, 25, dict(robots_per_world=8, side=6.0))], H=52, batch=128,
                         ckpt='stage2.pth', noise=False, localization=LOCALIZATION),
    # stage 1 with 2 straight drivers per world: H (N - 4) = 1760 kept rows are 6.9 minibatches of 256
    'masked_stage1': dict(stage=1, comps=[('stage1', 2, 1, 19, {})], H=40, batch=256, ckpt='stage1_2.pth', noise=False,
                          non_cooperative=(2, 0.8)),
    # the mix with every link of the chain on and a crowd that sees the map
    'chain': dict(stage=2, comps=MIX, H=52, batch=256, ckpt='stage2.pth', noise=True, latency=LATENCY,
                  dynamics=DYNAMICS, localization=dict(LOCALIZATION, seed=CHAIN_SEED), crowd=2),
    # arena worlds re-laid inside the horizon and across it; robots parked until their world's last episode ends
    'arena': dict(stage=2, comps=[ARENA], H=52, batch=128, ckpt='stage2.pth', noise=False),
    # stage 1's shape on its map with a pillar, steered and rewarded by the geodesic planner: every re-spawn re-plans, episodes end on tick
    # 39 = H - 1 and others straddle the boundary, their returns corrected in update 2
    'planner_stage1': dict(stage=1, comps=[('stage1', 2, 1, 19, dict(map_=_stage1_pillar))], H=40, batch=256,
                           ckpt='stage1_2.pth', noise=False, planner='geodesic'),
    # the arena case steered by waypoints, with the tick's own rewards
    'planner_straight': dict(stage=2, comps=[ARENA], H=52, batch=128, ckpt='stage2.pth', noise=False,
                             planner='straight'),
    # stage 2 | arena with every link of the chain the planner accepts (localization error it refuses), the planner
    # last; a 28-tick arena time-out, so that arena episodes straddle the boundary
    'planner_chain': dict(stage=2, comps=[('stage2', 1, 2, 25, {}), ARENA[:3] + (28,) + ARENA[4:]], H=52, batch=256,
                          ckpt='stage2.pth', noise=True, latency=LATENCY, dynamics=DYNAMICS, crowd=2,
                          planner='geodesic'),
}
SEED = 3


def _scenario(name, timeout, extra):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    sc = make_scenario(name, **{k: v() if callable(v) else v for k, v in extra.items()})
    return dataclasses.replace(sc, timeout=timeout)


class _Lines(logging.Handler):
    def __init__(self):
        super().__init__()
        self.records = []

    def emit(self, record):
        self.records.append(record.msg if not isinstance(record.msg, str) else record.getMessage())


def _np(t):
    return t.detach().cpu().numpy().copy()


# ------------------------------------------------------------------------------------------------ recording
class Recorder:
    def __init__(self, monkeypatch, policy, optimizer, generator, envs):
        from rl_collision_avoidance_b200 import noise as noise_mod
        from rl_collision_avoidance_b200 import trainer
        from rl_collision_avoidance_b200.crowd import Crowd
        from rl_collision_avoidance_b200.orca import NonCooperative
        from rl_collision_avoidance_b200.planner import Planner
        self.policy, self.opt, self.gen = policy, optimizer, generator
        self.ticks, self.fv, self.noise_cmds, self.gtd, self.updates = [], [], [], [], []
        self.executed = [[] for _ in envs]          # per component and tick: the command control_vel received
        self.overrides = [[] for _ in envs]         # per component and tick: the action after the masked override
        self.plans = [[] for _ in envs]             # per component, the start's then each tick's Planner.update: the
                                                    # status and psi_prev (psi) it left
        self.ro = self.comps = self.stats = None
        rec = self

        compose0 = trainer.compose

        def compose(envs, ro, noise=None, latency=None, dynamics=None, localization=None):
            rec.ro = ro
            rec.comps = compose0(envs, ro, noise, latency, dynamics, localization)
            return rec.comps
        monkeypatch.setattr(trainer, 'compose', compose)

        def index(env):
            return next(k for k, e in enumerate(envs) if e is env)

        for k, e in enumerate(envs):
            def control_vel(action, *args, _cv0=e.control_vel, _k=k, **kw):
                rec.executed[_k].append(action.detach().clone())
                return _cv0(action, *args, **kw)
            monkeypatch.setattr(e, 'control_vel', control_vel)

        for cls in (Crowd, NonCooperative):
            def apply(self_, action, _apply0=cls.apply):
                out = _apply0(self_, action)
                rec.overrides[index(self_.env)].append(out.clone())
                return out
            monkeypatch.setattr(cls, 'apply', apply)

        up0 = Planner.update

        def update(self_, flags=None, reward=None, eplog=None, gs=None):
            out = up0(self_, flags, reward, eplog, gs)
            rec.plans[index(self_.env)].append(dict(status=self_.status().clone(),
                                                    psi=None if self_.psi_prev is None else self_.psi_prev.clone()))
            return out
        monkeypatch.setattr(Planner, 'update', update)

        fv0 = policy.forward_values

        def forward_values(x, gs, v_out=None, mean_out=None):
            v, mean = fv0(x, gs, v_out, mean_out)
            rec.fv.append((x.data_ptr(), v.clone(), mean.clone()))
            return v, mean
        monkeypatch.setattr(policy, 'forward_values', forward_values)

        ga0 = trainer.generate_action

        def generate_action(env, state_list, policy, action_bound, out=None):
            r = ga0(env=env, state_list=state_list, policy=policy, action_bound=action_bound, out=out)
            slot = (state_list[0].data_ptr() - rec.ro.stacks.data_ptr()) // rec.ro.stacks[0].nbytes
            rec.ticks.append(dict(slot=slot, seed=policy.sample_seed, counter=policy.sample_counter,
                                  mean=rec.fv[-1][2], scaled=r[3].clone()))
            return r
        monkeypatch.setattr(trainer, 'generate_action', generate_action)

        act0 = noise_mod.Noise.action

        def action(self_, scaled):
            draw = self_.action_draws
            out = act0(self_, scaled)
            rec.noise_cmds.append((self_.stream_id, draw, scaled.clone(), out.clone()))
            return out
        monkeypatch.setattr(noise_mod.Noise, 'action', action)

        gtd0 = trainer.generate_train_data

        def generate_train_data(rewards, gamma, values, last_value, dones, lam):
            tg, adv = gtd0(rewards=rewards, gamma=gamma, values=values, last_value=last_value, dones=dones, lam=lam)
            rec.gtd.append(dict(rewards=_np(rewards), values=_np(values), last_value=_np(last_value), dones=_np(dones),
                                gamma=gamma, lam=lam, targets=_np(tg), advs=_np(adv)))
            return tg, adv
        monkeypatch.setattr(trainer, 'generate_train_data', generate_train_data)

        def wrap_update(f0):
            def update(**kw):
                ro = rec.ro
                u = dict(snap={k: _np(getattr(ro, k)) for k in ('stacks', 'gs', 'actions', 'logprobs', 'values',
                                                                 'rewards', 'flags', 'eplog')},
                         filter_index=list(kw.get('filter_index') or []), flat=rec.policy.flat.clone(),
                         m=rec.opt.exp_avg.clone(), v=rec.opt.exp_avg_sq.clone(), steps=[],
                         gen_state=rec.gen.get_state(), step_count=rec.opt.step_count,
                         ticks=rec.ticks[-ro.actions.shape[0]:])
                rec.updates.append(u)
                u['rows'] = f0(**kw)
                return u['rows']
            return update
        monkeypatch.setattr(trainer, 'ppo_update_stage1', wrap_update(trainer.ppo_update_stage1))
        monkeypatch.setattr(trainer, 'ppo_update_stage2', wrap_update(trainer.ppo_update_stage2))

        step0 = optimizer.step

        def step(grad_scale=1.0):
            p = rec.policy
            before = dict(p=p.flat.clone(), g=p.grad.clone(), m=optimizer.exp_avg.clone(),
                          v=optimizer.exp_avg_sq.clone(),
                          t=optimizer.step_count + 1, grad_scale=grad_scale)
            step0(grad_scale=grad_scale)
            before.update(p1=p.flat.clone(), m1=optimizer.exp_avg.clone(), v1=optimizer.exp_avg_sq.clone())
            rec.updates[-1]['steps'].append(before)
        monkeypatch.setattr(optimizer, 'step', step)


def _perturbations(c):
    """The perturbation settings of case c: noise, latency, dynamics and localization params (or None), the masked
    agents ('crowd', k, CrowdParams) / ('non_cooperative', k, speed) (or None) and the planner (or None)."""
    from rl_collision_avoidance_b200.crowd import CrowdParams
    from rl_collision_avoidance_b200.dynamics import DynamicsParams
    from rl_collision_avoidance_b200.latency import LatencyParams
    from rl_collision_avoidance_b200.localization import LocalizationParams
    from rl_collision_avoidance_b200.noise import NoiseParams
    masked = None
    if 'crowd' in c:
        masked = ('crowd', c['crowd'], CrowdParams())
    elif 'non_cooperative' in c:
        masked = ('non_cooperative',) + tuple(c['non_cooperative'])
    return dict(noise=NoiseParams(**NOISE) if c['noise'] else None,
                latency=LatencyParams(**c['latency']) if 'latency' in c else None,
                dynamics=DynamicsParams(**c['dynamics']) if 'dynamics' in c else None,
                localization=LocalizationParams(**c['localization']) if 'localization' in c else None,
                masked=masked, planner=c.get('planner'))


def _train(case, monkeypatch):
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from rl_collision_avoidance_b200.trainer import run
    c = CASES[case]
    envs, scs = [], []
    for name, W, ar, timeout, extra in c['comps']:
        sc = _scenario(name, timeout, extra)
        scs.append((sc, W, ar))
        envs.append(StageWorld(512, scenario=sc, num_worlds=W, seed=SEED, auto_reset=ar))
    N = sum(e.N for e in envs)
    policy = CNNPolicy(frames=3, action_space=2, seed=SEED, max_batch=max(c['batch'], N))
    policy.load_state_dict(torch.load(os.path.join(CKPT, c['ckpt']), map_location='cuda'))
    opt = Adam(policy.parameters(), lr=LR)
    gen = torch.Generator(device='cuda').manual_seed(SEED)
    hp = dict(HORIZON=c['H'], GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=c['batch'], EPOCH=2, COEFF_ENTROPY=COEFF,
              CLIP_VALUE=CLIP, NUM_ENV=N, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    pt = _perturbations(c)
    masked = pt['masked']
    rec = Recorder(monkeypatch, policy, opt, gen, envs)
    lg, lc = logging.getLogger(f'replay_{case}'), logging.getLogger(f'replay_cal_{case}')
    hl, hc = _Lines(), _Lines()
    for l, h in ((lg, hl), (lc, hc)):
        l.setLevel(logging.INFO)
        l.propagate = False
        l.addHandler(h)
    try:
        rec.stats = run(env=envs if len(envs) > 1 else envs[0], policy=policy, policy_path=None,
                        action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp, logger=lg, logger_cal=lc,
                        stage=c['stage'], max_updates=2, generator=gen, noise=pt['noise'], latency=pt['latency'],
                        dynamics=pt['dynamics'], localization=pt['localization'],
                        non_cooperative=masked[1:] if masked and masked[0] == 'non_cooperative' else None,
                        crowd=(masked[1], masked[2], True) if masked and masked[0] == 'crowd' else None,
                        planner=pt['planner'])
    finally:
        lg.removeHandler(hl)
        lc.removeHandler(hc)
    torch.cuda.synchronize()
    return rec, envs, scs, pt, hl.records, hc.records


# ------------------------------------------------------------------------------------------------ a. environment
class PlanReplay:
    """The planner of one component restated from planner_ref alone: build_plan_tables' graph, each row's goal entry
    (ref.goal_entry) re-planned by scipy's Dijkstra when it changes (ref.Graphs), the row's status and waypoint
    (ref.waypoint) and psi (planner_reward_ref) on the oracle's pose and goal, then with 'geodesic' the shaped reward
    and the episodes' shaping.  `plans` are the device's records of the component (Recorder.plans): the status and psi
    each Planner.update left, the start's first."""

    def __init__(self, kind, sc, cfg, plans, n):
        from rl_collision_avoidance_b200.planner import build_plan_tables
        t = build_plan_tables(sc.map)
        self.kind, self.m, self.label, self.graphs = kind, sc.map, t.label, planner_ref.Graphs(t.label, t.rects)
        self.ppm, self.res, self.gain = (float(np.float32(x)) for x in (cfg.ppm, cfg.resolution, cfg.progress_gain))
        self.plans = plans
        self.entry = [False] * n                     # the goal entry each row's field was planned for (None: no entry)
        self.field = [None] * n                      # (rect, D) of the row's field
        self.count = np.zeros(3, np.int64)           # the rows of each status since the update's stats were checked
        self.exempt = np.zeros(n, bool)              # rows whose waypoint the float64 walk may place elsewhere
        self.psi_prev = self.psi_start = None        # the device's psi after the last update / at the episode's start

    def update(self, i, pose, goal, gs_in, gs_dev, what, ev):
        """Planner.update number i (0: the run's start, g + 1: tick g) on the state the tick and any re-layout left:
        re-plan, then each row's status against the device's, its gs (gs_dev, what the policy read) against the
        waypoint's and psi against the float64 one.  Returns the gs the replay carries: the tick's where the goal is in
        sight or there is no plan, the device's checked waypoint gs elsewhere and on exempt rows."""
        m, ppm = self.m, self.ppm
        dev = self.plans[i]
        status, psi = _np(dev['status']), None if dev['psi'] is None else _np(dev['psi'])
        self.exempt[:] = False
        for a in range(len(pose)):
            e = planner_ref.goal_entry(self.label, m.origin_cx, m.origin_cy, ppm, goal[a, 0], goal[a, 1])
            if e != self.entry[a]:
                self.entry[a] = e
                self.field[a] = None if e is None else self.graphs.field(e)
                ev['replanned'] += int(e is not None)
            rect, D = self.field[a] or (None, None)
            w = planner_ref.waypoint(self.label, m.origin_cx, m.origin_cy, ppm, self.res, D, rect, e is not None,
                                     pose[a], goal[a])
            s = int(status[a])
            if s != 1:
                assert _bits_equal(gs_dev[a], gs_in[a]), f'{what} row {a}: status {s} and another gs than the tick\'s'
            ok = s == w[0]
            if ok and s == 1:
                dx, dy = w[1][0] - float(pose[a, 0]), w[1][1] - float(pose[a, 1])
                c, sn = math.cos(float(pose[a, 2])), math.sin(float(pose[a, 2]))
                ok = abs(dx * c + dy * sn - gs_dev[a, 0]) < 1e-4 and abs(dy * c - dx * sn - gs_dev[a, 1]) < 1e-4
                assert _bits_equal(gs_dev[a, 2:], gs_in[a, 2:]), f'{what} row {a}: the waypoint gs\'s speed'
            if not ok:
                # allowed only where a tested segment passes within 1e-5 m of a cell corner (test_planner)
                u, v = float(pose[a, 0]) * ppm, float(pose[a, 1]) * ppm
                near = planner_ref.corner_dist(u, v, float(goal[a, 0]) * ppm, float(goal[a, 1]) * ppm) < 1e-5 * ppm
                for (x, y) in (w[2] or []):
                    near |= planner_ref.corner_dist(u, v, x - m.origin_cx + 0.5, y - m.origin_cy + 0.5) < 1e-5 * ppm
                assert near, f'{what} row {a}: status {s}, waypoint gs {gs_dev[a]}; float64 status {w[0]} at {w[1]}'
                self.exempt[a] = True
            elif psi is not None:
                want = rref.psi_of(w, self.res, D, rect, pose[a])
                assert abs(float(psi[a]) - want) <= psi_bound(psi[a], pose[a, 3]), \
                    f'{what} row {a}: psi {psi[a]!r}, float64 {want!r}'
                ev['psi_checked'] += 1
            self.count[s] += 1
            ev[f'status_{s}'] += 1
        ev['plan_rows'] += len(pose)
        ev['exempt'] += int(self.exempt.sum())
        if i == 0 and psi is not None:
            self.psi_prev, self.psi_start = psi, psi.copy()       # every row starts an episode
        return np.where((status == 1)[:, None], gs_dev, gs_in)

    def shape(self, i, flags, reward, reward_dev, what, ev):
        """With 'geodesic', after update(i): the device's reward against the tick's plus gain (psi_prev - psi) on a
        non-terminal tick (rref.shaped_reward, test_planner_reward's bound, from the device's psi checked in update) and
        the tick's bit for bit on a terminal one.  Returns the device's rewards, their float64 values and, per row, the
        shaping gain (psi_start - psi_prev) the return of an episode the tick ended gets; then psi_prev = psi and
        psi_start restarts where flags[:, 3] is set."""
        psi = _np(self.plans[i]['psi'])
        r64 = reward.astype(np.float64)
        for a in range(len(reward)):
            if flags[a, 0] != 0:
                assert _bits_equal(reward_dev[a], reward[a]), f'{what} row {a}: terminal reward {reward_dev[a]!r} ' \
                                                              f'is not the tick\'s {reward[a]!r}'
                continue
            r64[a] = rref.shaped_reward(reward[a], flags[a], self.psi_prev[a], psi[a], self.gain)
            term = self.gain * (float(self.psi_prev[a]) - float(psi[a]))
            assert abs(float(reward_dev[a]) - r64[a]) <= shaped_bound(reward[a], term), \
                f'{what} row {a}: shaped reward {reward_dev[a]!r}, float64 {r64[a]!r}'
            ev['shaped_changed'] += int(reward_dev[a] != reward[a])
        corr = self.gain * (self.psi_start.astype(np.float64) - self.psi_prev.astype(np.float64))
        self.psi_prev = psi
        restart = flags[:, 3] != 0
        self.psi_start[restart] = psi[restart]
        return reward_dev.copy(), r64, corr


class OracleComponent:
    """The CPU oracle of one component, the restated scan deque and the episode bookkeeping of its robots."""

    def __init__(self, k, comp, sc, W, ar, pt, plans):
        from oracle.oracle import OracleWorld, OrcConfig
        from rl_collision_avoidance_b200.noise import scan_host
        from rl_collision_avoidance_b200.orca import ObstacleSet
        from rl_collision_avoidance_b200.scenarios import ArenaLayout, arena_layout_host, fill_config, \
            random_layout_host
        self.k, self.c, self.sc, self.noise = k, comp, sc, pt['noise']
        self.cfg = cfg = comp.env.cfg                # the product's config struct, for the host twins
        ocfg = fill_config(OrcConfig(), sc, num_worlds=W, beams=512, auto_reset=ar, seed=SEED)
        o = self.o = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
        self.relayout = sc.layout is not None
        self.arena = isinstance(sc.layout, ArenaLayout)
        o.reset_world()
        o.reset_pose()
        o.generate_goal_point()
        if self.relayout:
            # the first layout: the random one, or the arena layout with the layout's own pick
            first = arena_layout_host if self.arena else random_layout_host
            o.pose[...], o.goal[...], o.acc[...], status = first(self.cfg, sc.layout, o.pose, o.goal, o.acc)
            assert not status.any()
            o.observe()
        n = o.N
        R, off = int(cfg.robots_per_world), int(cfg.world_offset)
        # the chain's restatements, stream k as compose gives component k
        lp, dp, zp = pt['latency'], pt['dynamics'], pt['localization']
        self.lat = None if lp is None else latency_ref.Latency(R, W, lp.scan_delay, lp.command_delay, lp.seed, off, k)
        self.dyn = None if dp is None else dynamics_ref.Dynamics(R, W, dp.linear, dp.angular, dp.seed,
                                                                 (cfg.v_min, cfg.v_max, cfg.w_min, cfg.w_max), cfg.dt,
                                                                 off, k)
        self.loc = None if zp is None else localization_ref.Localization(
            R, W, zp.pose_sigma, zp.heading_sigma, zp.correlation_time, zp.speed_sigma, zp.seed, cfg.dt, off, k)
        self.masked = pt['masked']
        self.mask = np.zeros(n, np.uint8)            # robots floor(j R / k), j < k, of every world (§9h, §9t)
        self.obstacles = self.segments = None
        if self.masked is not None:
            kk = self.masked[1]
            for w in range(W):
                self.mask[w * R + np.arange(kk) * R // kk] = 1
            if self.masked[0] == 'crowd':
                self.obstacles = ObstacleSet(cfg, sc.map.cells, self.masked[2].wall_dist)
                self.segments = self.obstacles.segments()[0]
        self.prev = None                             # the flags of the tick before, None before the run's first
        self.live = np.ones(n, np.uint8)
        self.stacks = ref.Stacks(o.obs)
        arr = self.stacks.array()
        if self.lat is not None:
            self.lat.scan(arr)                       # every row starts an episode: its stack is left as it is
        if self.noise is not None:
            arr = scan_host(self.cfg, self.noise, 0, arr, None, stream_id=k)
        self.stacks.load(arr)
        self.scan_draws = 1
        self.gs = o.gs.copy()
        if self.loc is not None:
            self.gs = self.loc.observe(o.pose, o.goal, self.gs, None)
        self.believed = (self.gs != o.gs).any(1)     # rows whose gs is not the true one
        # episode bookkeeping (ppo_stage1.py:51-57, 127-131; ppo_stage2.py:49-56, 136-137)
        self.episode = np.zeros(n, np.int64)
        self.steps = np.zeros(n, np.int64)
        self.ep_reward = np.zeros(n)
        self.ep_abs = np.zeros(n)
        self.goal = o.goal[:, 0:2].copy()
        self.init = o.pose[:, 0:2].copy()
        self.idle = np.zeros(n, bool)                 # stage 2's liveflag false / a parked random robot
        self.last_r = np.zeros(n, np.float32)
        self.ep_sabs = np.zeros(n)                    # sum of |shaped reward| in float64, for the float64 sum's rounding
        self.ep_update = np.zeros(n, np.int64)        # the update an episode started in
        self.plan = None if pt['planner'] is None else PlanReplay(pt['planner'], sc, cfg, plans, n)

    def start_plan(self, gs_dev, ev):
        """The planner's update at the run's start, against slot 0 of update 0 (gs_dev)."""
        if self.plan is not None:
            self.gs = self.plan.update(0, self.o.pose, self.o.goal, self.gs, gs_dev, f'start {self.c.name}', ev)

    def state(self):
        return self.stacks.array(), self.gs.copy()

    def command(self, scaled, g, rec, ev):
        """The command executed on global tick g for the sampled `scaled` rows: masked override -> latency -> noise ->
        limits, the last two links with the flags of the tick before; each recorded link is held to it bit for bit and
        the result to what control_vel received."""
        from rl_collision_avoidance_b200.noise import action_host
        o, what = self.o, f'tick {g} {self.c.name}'
        cmd = scaled
        if self.masked is not None:
            if self.masked[0] == 'crowd':
                from rl_collision_avoidance_b200.crowd import crowd_host
                want = crowd_host(self.cfg, o.pose, o.goal, o.meta, self.mask, cmd, self.masked[2],
                                  obstacles=self.obstacles)
            else:
                from rl_collision_avoidance_b200.orca import noncoop_host
                want = noncoop_host(self.cfg, o.pose, o.goal, o.meta, self.mask, cmd, speed=self.masked[2])
            assert _bits_equal(_np(rec.overrides[self.k][g]), want), f'{what}: masked override'
            self._check_masked(want, ev)
            ev['masked_changed'] += int((want != cmd).any(1).sum())
            cmd = want
        if self.lat is not None:
            out = self.lat.action(cmd, self.prev)
            ev['command_delayed'] += int((out != cmd).any(1).sum())
            cmd = out
        if self.noise is not None and self.noise.action_on:
            sid, draw, inp, out = [x for x in rec.noise_cmds if x[0] == self.k][g]
            assert draw == g and _bits_equal(_np(inp), cmd), f'{what}: the noised command\'s input'
            want = action_host(self.cfg, self.noise, g, cmd, stream_id=self.k)
            assert _bits_equal(_np(out), want), f'{what}: noised command'
            ev['noised_rows'] += int((want != cmd).any(1).sum())
            cmd = want
        if self.dyn is not None:
            vel = self.dyn.vel.copy()
            out = self.dyn.action(cmd, self.prev)
            v0, v1, w0, w1 = self.dyn.bounds
            target = np.stack([dynamics_ref.target(cmd[:, 0], v0, v1), dynamics_ref.target(cmd[:, 1], w0, w1)], 1)
            ev['limited'] += int((out != cmd).any(1).sum())
            ev['clamped'] += int((out != target).sum())
            if self.prev is not None:
                crashed = (self.prev[:, 1] != 0) & (self.prev[:, 3] == 0)
                ev['crash_prev_reset'] += int((crashed & vel.any(1)).sum())
            cmd = out
        assert _bits_equal(_np(rec.executed[self.k][g]), cmd), f'{what}: the command control_vel received'
        return cmd

    def _check_masked(self, act, ev):
        """the twin's masked rows against the float64 restatements: crowd_ref within test_crowd's bound (agents with a
        distance within 1e-4 of a cut-off left out, as there), the straight driver within test_noncoop's"""
        from rl_collision_avoidance_b200.orca import DEFAULTS
        o, cfg = self.o, self.cfg
        R = int(cfg.robots_per_world)
        for a in np.flatnonzero(self.mask):
            if self.masked[0] == 'crowd':
                p = self.masked[2]
                segs = _segments_near(self.segments, o.pose[a, 0:2].astype(np.float64), p.wall_dist + 0.01)
                d = crowd_ref.distances(cfg, o.pose, a, segs)
                near = np.concatenate((d[:R - 1] - p.neighbour_dist, d[R - 1:] - p.wall_dist))
                if ((np.abs(near) < 1e-4) & (near != 0)).any():
                    continue
                want, tol = crowd_ref.crowd_action(cfg, o.pose, o.goal, o.meta, self.mask, a, p, segs), CROWD_TOL
            else:
                pos, th, _ = orca_ref.agent_state(o.pose, o.goal, o.meta)
                speed = float(self.masked[2])
                v = orca_ref.preferred(pos[a], o.goal[a, 0:2], speed, float(cfg.dt))
                want, tol = orca_ref.track(th[a], v, speed, cfg.w_min, cfg.w_max, DEFAULTS['heading_gain']), \
                    NONCOOP_TOL
            assert np.abs(act[a] - want).max() <= tol, (self.c.name, a, act[a], want)
            ev['masked_checked'] += 1

    def tick(self, cmd, g, ev, dev):
        """one tick at global tick g of update dev['u']: reward, flags, eplog, the rows that were idle on it and those
        that ended.  dev holds the device's gs, reward and eplog of the tick: with a planner the replay checks them and
        carries the device's where it may not restate them bit for bit."""
        from rl_collision_avoidance_b200.noise import scan_host
        from rl_collision_avoidance_b200.scenarios import arena_relayout_host, relayout_host
        o = self.o
        idle = self.idle | (self.live == 0)
        o.step(cmd, live=self.live if self.relayout else None)
        reward, flags, eplog = o.reward.copy(), o.flags.copy(), o.eplog.copy()
        obs, gs = o.obs.copy(), o.gs.copy()
        ended = (flags[:, 0] != 0) & ~idle
        restart = flags[:, 3] != 0
        self.stacks.tick(obs, restart)
        if self.relayout:
            relay = arena_relayout_host if self.arena else relayout_host
            o.pose[...], o.goal[...], o.acc[...], o.meta[...], flags, self.live, status = relay(
                self.cfg, self.sc.layout, o.pose, o.goal, o.acc, o.meta, flags)
            assert not status.any()
            o.observe()
            relaid = flags[:, 3] != 0
            arr = self.stacks.array()
            arr[relaid] = o.obs[relaid][:, None, :]
            self.stacks.load(arr)
            gs[relaid] = o.gs[relaid]
            restart = relaid
        arr = self.stacks.array()
        if self.lat is not None:
            newest = arr[:, 2].copy()
            self.lat.scan(arr, flags)
            ev['scan_delayed'] += int((arr[:, 2] != newest).any(1).sum())
        if self.noise is not None:
            newest = arr[:, 2].copy()
            arr = scan_host(self.cfg, self.noise, self.scan_draws, arr, flags, stream_id=self.k)
            ev['noised_scans'] += int((arr[:, 2] != newest).any(1).sum())
        self.stacks.load(arr)
        self.scan_draws += 1
        if self.loc is not None:
            # on the oracle's pose and goal after the re-layout, with this tick's flags
            sigma = self.loc.sigma.copy()
            believed = self.loc.observe(o.pose, o.goal, gs, flags)
            fresh = flags[:, 3] != 0
            ev['sigma_redrawn' if not self.relayout else 'relaid_sigma_redrawn'] += int(
                (fresh & (self.loc.sigma != sigma).any(1)).sum())
            self.believed = (believed != gs).any(1)
            ev['believed'] += int(self.believed.sum())
            gs = believed
        # the planner last, on the state and flags the re-layout left
        tick_reward, r64, corr = reward, reward.astype(np.float64), None
        what = f'update {dev["u"]} tick {g} {self.c.name}'
        if self.plan is not None:
            gs = self.plan.update(g + 1, o.pose, o.goal, gs, dev['gs'], what, ev)
            if self.plan.kind == 'geodesic':
                reward, r64, corr = self.plan.shape(g + 1, flags, reward, dev['reward'], what, ev)
        self.gs = gs
        self.prev = flags
        # bookkeeping
        lines = []
        live_now = ~idle
        self.steps[live_now] += 1
        self.ep_reward[live_now] += r64[live_now]
        self.ep_abs[live_now] += np.abs(tick_reward[live_now].astype(np.float64))
        self.ep_sabs[live_now] += np.abs(r64[live_now])
        for i in np.nonzero(ended)[0]:
            # the tick's return is a float32 running sum of `steps` terms: within steps u sum |r| of the float64 sum
            tol = self.steps[i] * U * self.ep_abs[i]
            if corr is not None:
                # the planner adds c = gain (psi_start - psi_prev) to it: E = fl(R + fl(gain fl(psi_start - psi_prev)))
                # with R the tick's return.  The two inner roundings put fl(...) within (2u + u^2) |c| of c, the
                # addition E within u |E| (1 + u) of R + fl(...); the float64 sum of the shaped rewards is R's float64
                # sum plus c (the shaping terms of the non-terminal ticks telescope to c), up to its own rounding, <=
                # steps 2^-52 sum |shaped reward|
                E, c = float(dev['eplog'][i, 2]), float(corr[i])
                tol += (2 * U + U * U) * abs(c) + U * (1 + U) * abs(E) + self.steps[i] * 2.0 ** -52 * self.ep_sabs[i]
                assert _bits_equal(np.delete(dev['eplog'][i], 2), np.delete(eplog[i], 2)), \
                    f'{what} row {i}: eplog columns but the return'
                assert abs(E - self.ep_reward[i]) <= tol + 1e-30, \
                    f'{what} row {i}: return {E!r}, float64 sum of the shaped rewards {self.ep_reward[i]!r}, bound {tol}'
                eplog[i, 2] = dev['eplog'][i, 2]
                ev['corrected'] += int(c != 0)
                ev['straddled'] += int(dev['u'] == 1 and self.ep_update[i] == 0)
            lines.append((i, self.episode[i], self.steps[i], self.ep_reward[i], tol, self.goal[i].copy(),
                          self.init[i].copy(), int(flags[i, 2])))
        self.idle = (self.idle | ended) & ~restart
        for i in np.nonzero(restart)[0]:
            self.episode[i] += 1
            self.steps[i] = 0
            self.ep_reward[i] = self.ep_abs[i] = self.ep_sabs[i] = 0.0
            self.ep_update[i] = dev['u'] if g % dev['H'] != dev['H'] - 1 else dev['u'] + 1
            self.goal[i] = o.goal[i, 0:2]
            self.init[i] = o.pose[i, 0:2]
        out = dict(reward=reward, flags=flags, eplog=eplog, idle=idle, ended=ended, lines=lines,
                   last_r=self.last_r.copy())
        self.last_r = reward.copy()
        return out


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _segments_near(segments, p, dist):
    """The segments (S, 4) within `dist` of the point p: crowd_ref walks every segment in Python, and one farther than
    wall_dist neither pushes the agent nor lies near its cut-off"""
    s = np.asarray(segments, np.float64).reshape(-1, 4)
    a, e = s[:, 0:2], s[:, 2:4] - s[:, 0:2]
    t = np.clip(((p - a) * e).sum(1) / np.maximum((e * e).sum(1), 1e-300), 0.0, 1.0)
    return s[np.hypot(*(p - a - t[:, None] * e).T) < dist]


def _episode_stats(ep):
    """episodes, success and crash rates (result 1 and 2) and the mean reward of the eplog rows ep (E, 8) float32,
    in their order; NaN without episodes"""
    n = len(ep)
    return {'episodes': n, 'success_rate': float(np.mean(ep[:, 6] == 1)) if n else math.nan,
            'crash_rate': float(np.mean(ep[:, 6] == 2)) if n else math.nan,
            'mean_ep_reward': float(ep[:, 2].mean()) if n else math.nan}


def _same(a, b):
    """a == b, NaN equal to NaN, through dicts"""
    if isinstance(a, dict) or isinstance(b, dict):
        return isinstance(a, dict) and isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return a == b or (isinstance(a, float) and isinstance(b, float) and math.isnan(a) and math.isnan(b))


def _masked_rows_across_boundaries(fd, starts, col_mask, H, N):
    """The masked rows t N + a of a component's first column a (`starts`) that continue a run of filtered rows from
    the previous component's last column, t N + a - 1, which get_filter_index (`fd`) filtered: a run of the united
    filter that crosses a component boundary with its masked part on one side."""
    fd = set(fd)
    return sum(1 for a in starts if col_mask[a] for t in range(H) if t * N + a - 1 in fd)


# ------------------------------------------------------------------------------------------------ float64 pieces
def _params64(policy, flat):
    from rl_collision_avoidance_b200.model.net import TENSORS
    out = {}
    for i, (name, shape) in enumerate(TENSORS):
        o = policy.offsets[i]
        out[name] = flat[o:o + math.prod(shape)].view(shape).double().clone()
    return out


def _forward64(P, x, gs, chunk=1024):
    """float64 value (n,), mean (n, 2) and, per row and head, the magnitude of the actor head's terms
    sum_k |w_k h_k| + |b| (n, 2): check_forward's mean bound (1e-5) holds for the synthetic weights of learner_ref; the
    checkpoints' heads sum larger terms, so the mean is held to the value's relative bound, 2e-5 of that magnitude
    (sigmoid and tanh have slope <= 1), and never below 1e-5"""
    vs, ms, zs = [], [], []
    W = torch.cat((P['actor1.weight'], P['actor2.weight'])).abs()
    b = torch.cat((P['actor1.bias'], P['actor2.bias'])).abs()
    with torch.no_grad():
        for r0 in range(0, x.shape[0], chunk):
            pre = []
            v, m, _ = ref_forward(P, x[r0:r0 + chunk].double(), gs[r0:r0 + chunk].double(), pre)
            h = torch.relu(dict(pre)['act_fc2'])
            vs.append(v)
            ms.append(m)
            zs.append(h @ W.T + b)
    return torch.cat(vs), torch.cat(ms), torch.cat(zs)


def _mean_bound(P, pre):
    """the bound on the device's mean per row and head (n, 2): see _forward64"""
    W = torch.cat((P['actor1.weight'], P['actor2.weight'])).detach().abs()
    b = torch.cat((P['actor1.bias'], P['actor2.bias'])).detach().abs()
    h = torch.relu(dict(pre)['act_fc2'].detach())
    return torch.clamp(2e-5 * (h @ W.T + b), min=1e-5)


ADV_U = 4 * U             # the device's normalised advantage: (x - mean) / std in float32, from float64 moments
ACTOR_SIDE = ('act_', 'actor', 'logstd')
CRITIC_SIDE = ('crt_', 'critic')


def _flip_rows_grad(policy, st, ii, x, gsx, act_all, lp_all, adv_n, tgt_all, pre, tower):
    """The float64 gradient of the minibatch loss's share from the rows with an undecided fc1 / fc2 ReLU mask in
    `tower` (a pre-activation within learner_ref.MARGIN of its layer's max of zero), or None when there is none.  A
    flipped mask changes only its own row's contribution to the sum over the minibatch, so the device's gradient may
    differ from float64 by up to twice that share."""
    rows = torch.zeros(len(ii), dtype=torch.bool, device=ii.device)
    for layer, z in pre:
        if layer in (tower + '_fc1', tower + '_fc2'):
            rows |= (z.detach().abs() < MARGIN * float(z.detach().abs().max())).any(1)
    if not rows.any():
        return None
    with torch.enable_grad():
        P = {n: t.requires_grad_(True) for n, t in _params64(policy, st['p']).items()}
        jj = ii[rows]
        v, mean, _ = ref_forward(P, x[jj].double(), gsx[jj].double())
        (pl, vl, _), _ = ref_losses(P, v, mean, act_all[jj], lp_all[jj], adv_n[jj], tgt_all[jj])
        ((pl + VCOEF * vl) * (len(jj) / len(ii))).backward()
    return {n: t.grad for n, t in P.items()}


def step_checks(check, what, policy, st, row, ii, x, gsx, act_all, lp_all, adv_n, tgt_all, ev):
    """One optimizer step, teacher-forced from the device's parameters at the step (st['p']) on the minibatch rows ii
    of the replayed schedule.

    Loss row.  The float64 losses (learner_ref.ref_losses) differ from the device's through the device's forward
    (its value within dv = 2e-5 max(1, |v|), check_forward's bound; its mean within dm, _mean_bound) and through the
    float32 loss reduction (check_step's 1e-5 of the loss, at least 1e-7).  First order:
      policy: |d ratio| = ratio |d logprob| <= ratio sum_d |a - mean| / sigma^2 dm, the advantage within ADV_U, so
              the policy loss moves by <= mean(ratio (|adv| |d logprob| + ADV_U |adv|));
      value:  mean((v - tgt)^2) moves by <= mean(2 |v - tgt| dv + dv^2) (the targets are the device's own);
      entropy: a function of logstd alone.
    Gradients.  check_step's 5e-5 of the layer scale holds where the forward is within check_forward's bounds for
    |v| <= 1: the mean within 1e-5, the value within 2e-5.  A gradient is first order in the error of the output its
    loss term reads, so the actor side (its towers, heads and logstd) is held to 5e-5 times this minibatch's
    max(dm) / 1e-5 and the critic side to 5e-5 times dv / 2e-5.  A tower's conv tensors with an undecided conv mask
    are held to at least 3e-3 (module docstring); an undecided fc mask adds twice its rows' share (_flip_rows_grad).
    Adam.  ref.adam_step in float64 from the device's p, g, m, v and step, with the float32 betas the kernel receives,
    against the bound of adam_bounds."""
    P = {n: t.requires_grad_(True) for n, t in _params64(policy, st['p']).items()}
    pre = []
    v, mean, _ = ref_forward(P, x[ii].double(), gsx[ii].double(), pre)
    act, old_lp, adv, tgt = act_all[ii], lp_all[ii], adv_n[ii], tgt_all[ii]
    (pl, vl, ent), loss = ref_losses(P, v, mean, act, old_lp, adv, tgt)
    loss.backward()
    with torch.no_grad():
        ratio = torch.exp(ref_logprob(P, mean, act) - old_lp)
        near = ((ratio - (1 - CLIP)).abs() < MARGIN) | ((ratio - (1 + CLIP)).abs() < MARGIN)
        assert not near.any(), f'{what}: a PPO ratio within {MARGIN} of 1 +- clip: choose another seed'
        ev['clipped'] += int(((ratio < 1 - CLIP) | (ratio > 1 + CLIP)).sum())
        dm = _mean_bound(P, pre)
        dv = 2e-5 * max(1.0, maxabs(v))
        dlp = ((act - mean).abs() / torch.exp(2 * P['logstd']) * dm).sum(1)
        bounds = (float((ratio * adv.abs() * (dlp + ADV_U)).mean()) + 1e-5 * max(abs(float(pl)), 1e-2),
                  float((2 * (v - tgt).abs() * dv + dv * dv).mean()) + 1e-5 * max(abs(float(vl)), 1e-2),
                  1e-5 * max(abs(float(ent)), 1e-2))
        for i, name in enumerate(('policy', 'value', 'entropy')):
            check(f'{what} {name} loss', abs(row[i] - float((pl, vl, ent)[i])), bounds[i])
        undecided = {layer: int((z.abs() < MARGIN * float(z.abs().max())).sum()) for layer, z in pre}
        factor = float(dm.max()) / 1e-5
        ev['worst_mean_factor'] = max(ev['worst_mean_factor'], factor)
        ev['worst_value_factor'] = max(ev['worst_value_factor'], dv / 2e-5)
        grads = {n: t.grad for n, t in P.items()}
        gdev = _params64(policy, st['g'])
        for tower in ('act', 'crt'):
            ev['undecided_conv'] += int(bool(undecided[tower + '_cv1'] or undecided[tower + '_cv2']))
            ev['undecided_fc'] += int(bool(undecided[tower + '_fc1'] or undecided[tower + '_fc2']))
        flip = {side: _flip_rows_grad(policy, st, ii, x, gsx, act_all, lp_all, adv_n, tgt_all, pre, tower)
                for side, tower in ((ACTOR_SIDE, 'act'), (CRITIC_SIDE, 'crt'))}
        for name, r in grads.items():
            side = ACTOR_SIDE if name.startswith(ACTOR_SIDE) else CRITIC_SIDE
            tower = 'act' if side is ACTOR_SIDE else 'crt'
            conv = '_fea_cv' in name and (undecided[tower + '_cv1'] or undecided[tower + '_cv2'])
            tol = 5e-5 * (factor if side is ACTOR_SIDE else dv / 2e-5)
            tol = max(tol, 3e-3) if conv else tol
            extra = 2 * maxabs(flip[side][name]) if flip[side] is not None else 0.0
            check(f'{what} grad {name}', maxabs(gdev[name] - r), tol * layer_scale(grads, name) + extra)
    p0, g0, m0, v0 = (_np(st[key]).astype(np.float64) for key in ('p', 'g', 'm', 'v'))
    p64, m64, v64 = ref.adam_step(p0, g0, m0, v0, st['t'], LR, (B1, B2), 1e-8)
    p1, m1, v1 = (_np(st[key]).astype(np.float64) for key in ('p1', 'm1', 'v1'))
    bm, bv, bp = adam_bounds(p0, g0, m0, v0, p1, p64, st['t'])
    for name, got, want, bound in (('exp_avg', m1, m64, bm), ('exp_avg_sq', v1, v64, bv), ('parameters', p1, p64, bp)):
        r = np.abs(got - want) / bound
        i = int(np.argmax(r))
        check(f'{what} Adam {name} (error / bound; worst at {i}: p {p0[i]:.9g} g {g0[i]:.9g} m {m0[i]:.9g} '
              f'v {v0[i]:.9g} got {got[i]:.9g} want {want[i]:.9g})', float(r[i]), 1.0)


def adam_bounds(p0, g0, m0, v0, p1, p64, step):
    """Error model of the fused Adam step (csrc/rlca_policy.cu, adam_update_one) against ref.adam_step with the same
    float32 betas, u = 2^-24 the unit roundoff (every float32 rounding is within u of its result):
      m = fmaf(b1, m, (1 - b1) g): 1 - b1 is exact (Sterbenz); the product and the fma round once each:
          <= 2u (b1 |m| + (1 - b1) |g|);
      v = fmaf(b2, v, (1 - b2) g g): two products and the fma: <= 3u (b2 v + (1 - b2) g^2);
      the step d = lr / bc1 * m / (sqrtf(v) / sqrt(bc2) + eps) carries m's error relative to m (bm / |m|: large where
          b1 m and (1 - b1) g cancel, as they do when the gradient changes sign) and half of v's relative error (the
          square root); lr's float32 rounding and eight float32 operations add <= 9u, taken as 16u;
          bc1 = 1 - powf(b1, t) and bc2 = 1 - powf(b2, t) are formed in float32 on the host, and powf's error
          (<= 1 ulp, 2u) is amplified by the cancellation b^t / (1 - b^t): 2u k1 for bc1, u k2 for bc2 under the
          square root;
      p - d rounds to within half an ulp of the result.
    Returns the bounds on m, v and p."""
    k1 = B1 ** step / (1 - B1 ** step)
    k2 = B2 ** step / (1 - B2 ** step)
    bm = 2 * U * (B1 * np.abs(m0) + (1 - B1) * np.abs(g0)) + TINY
    bv = 3 * U * (B2 * v0 + (1 - B2) * g0 * g0) + TINY
    mv = np.abs(B1 * m0 + (1 - B1) * g0)
    vv = B2 * v0 + (1 - B2) * g0 * g0
    rel = (16 * U + 2 * U * k1 + U * k2 + np.divide(bm, mv, out=np.zeros_like(mv), where=mv > 0)
           + 0.5 * np.divide(bv, vv, out=np.zeros_like(vv), where=vv > 0))
    bp = 0.5 * np.spacing(np.abs(p1).astype(np.float32)).astype(np.float64) + rel * np.abs(p64 - p0) + TINY
    return bm, bv, bp


# ------------------------------------------------------------------------------------------------ the test
@pytest.mark.parametrize('case', list(CASES))
def test_trainer_replays_against_the_reference_loop(built, monkeypatch, case):
    t_start = time.perf_counter()
    c = CASES[case]
    stage, H = c['stage'], c['H']
    rec, envs, scs, pt, lines, cal = _train(case, monkeypatch)
    t_train = time.perf_counter() - t_start
    noise = pt['noise']
    policy = rec.policy
    comps = rec.comps
    N = sum(e.N for e in envs)
    assert len(rec.updates) == 2 and len(rec.gtd) == 2 and len(rec.ticks) == 2 * H and len(rec.stats) == 2
    assert all(len(x) == 2 * H for x in rec.executed)
    assert all(len(x) == (2 * H if pt['masked'] else 0) for x in rec.overrides)
    assert all(len(x) == (2 * H + 1 if pt['planner'] else 0) for x in rec.plans)
    oc = [OracleComponent(k, comp, sc, W, ar, pt, rec.plans[k])
          for k, (comp, (sc, W, ar)) in enumerate(zip(comps, scs))]
    col_mask = np.concatenate([o.mask for o in oc]) != 0
    col_comp = np.concatenate([np.full(o.o.N, k) for k, o in enumerate(oc)])
    check = Checks()
    ev = collections.defaultdict(int)
    for key in ('ended', 'ended_last_tick', 'idle', 'respawn', 'relaid', 'filtered', 'boundary_runs', 'noised_rows',
                'steps', 'clipped', 'undecided_conv', 'undecided_fc', 'worst_mean_factor', 'worst_value_factor'):
        ev[key] = 0
    for o in oc:
        o.start_plan(rec.updates[0]['snap']['gs'][0, o.c.a:o.c.b], ev)
    expected_lines = []
    for u, up in enumerate(rec.updates):
        snap = up['snap']
        believed = np.zeros((H, N), bool)           # rows whose gs slot t is not the true gs
        ended_rows = []                             # (t, column, eplog row) of the episodes that ended
        # ---- a. the environment, bit for bit, and the episode bookkeeping
        st0 = [o.state() for o in oc]
        for o, (s, g) in zip(oc, st0):
            a, b = o.c.a, o.c.b
            assert _bits_equal(snap['stacks'][0, a:b], s), f'update {u}: stacks[0] of {o.c.name} (carry-over)'
            assert _bits_equal(snap['gs'][0, a:b], g), f'update {u}: gs[0] of {o.c.name} (carry-over)'
        dones = np.zeros((H, N), bool)
        rewards = np.zeros((H, N), np.float32)
        upd_lines = []
        for t in range(H):
            g = u * H + t
            tk = up['ticks'][t]
            assert tk['slot'] == t, f'update {u} tick {t}: the policy read stack slot {tk["slot"]}'
            scaled = _np(tk['scaled'])
            for o in oc:
                a, b = o.c.a, o.c.b
                believed[t, a:b] = o.believed
                if u == 1 and t == 0 and o.lat is not None and o.lat.cr[1] > 0:
                    # rows whose episode ended on update 1's last tick restart their command rings here
                    ev['ring_restart_on_boundary'] += int((o.prev[:, 3] != 0).sum())
                dev = dict(u=u, H=H, gs=snap['gs'][t + 1, a:b], reward=snap['rewards'][t, a:b],
                           eplog=snap['eplog'][t, a:b])
                r = o.tick(o.command(scaled[a:b], g, rec, ev), g, ev, dev)
                s, gsn = o.state()
                what = f'update {u} tick {t} {o.c.name}'
                assert _bits_equal(snap['stacks'][t + 1, a:b], s), f'{what}: stack'
                assert _bits_equal(snap['gs'][t + 1, a:b], gsn), f'{what}: gs'
                assert _bits_equal(snap['rewards'][t, a:b], r['reward']), f'{what}: reward'
                assert _bits_equal(snap['flags'][t, a:b], r['flags']), f'{what}: flags'
                e = r['ended']
                assert _bits_equal(snap['eplog'][t, a:b][e], r['eplog'][e]), f'{what}: eplog of ended episodes'
                assert (r['flags'][e, 2] != 0).all(), f'{what}: an ended episode without a result'
                ended_rows += [(t, a + i, r['eplog'][i]) for i in np.flatnonzero(e)]
                # stage 2's liveflag: an idle robot's row repeats its last reward and stays terminal, result 0
                idle = r['idle']
                if idle.any():
                    assert _bits_equal(r['reward'][idle], r['last_r'][idle]), f'{what}: stale reward of idle rows'
                    assert (r['flags'][idle, 0] == 1).all() and (r['flags'][idle, 2] == 0).all(), f'{what}: idle flags'
                ev['idle'] += int(idle.sum())
                ev['ended'] += int(e.sum())
                ev['ended_last_tick'] += int(e.sum()) if t == H - 1 else 0
                ev['respawn' if not o.relayout else 'relaid'] += int((r['flags'][:, 3] != 0).sum())
                dones[t, a:b] = r['flags'][:, 0] != 0
                rewards[t, a:b] = r['reward']
                for (i, epi, steps, rsum, tol, goal, init, res) in r['lines']:
                    upd_lines.append((t, a + i, o, i, epi, steps, rsum, tol, goal, init, res))
        # ---- b. the policy per tick, at the weights of the update's start
        P = _params64(policy, up['flat'])
        logstd = _np(up['flat'][policy.offsets[0]:policy.offsets[0] + 2])
        x = torch.from_numpy(snap['stacks'][:H].reshape(H * N, 3, 512)).cuda()
        gsx = torch.from_numpy(snap['gs'][:H].reshape(H * N, 4)).cuda()
        v64, m64, zs = _forward64(P, x, gsx)
        mean_dev = torch.stack([tk['mean'] for tk in up['ticks']]).reshape(H * N, 2)
        vs = max(1.0, maxabs(v64))
        check(f'update {u} rollout value', maxabs(torch.from_numpy(snap['values']).cuda().reshape(-1).double() - v64),
              2e-5 * vs)
        check(f'update {u} rollout mean (error / bound)',
              float(((mean_dev.double() - m64).abs() / torch.clamp(2e-5 * zs, min=1e-5)).max()), 1.0)
        mean_np = _np(mean_dev).reshape(H, N, 2)
        wa, wl = 0.0, 0.0
        for t, tk in enumerate(up['ticks']):
            assert tk['seed'] == policy.sample_seed
            act64, z = sample_ref.sample(mean_np[t], logstd, tk['seed'], tk['counter'])
            act = snap['actions'][t]
            sz = sample_ref.sigma(logstd) * np.abs(z)
            wa = max(wa, float((np.abs(act - act64) / action_bound(act, sz)).max()))
            lp = sample_ref.log_prob(act, mean_np[t], logstd)
            wl = max(wl, float((np.abs(snap['logprobs'][t] - lp) / lp_bound(act, mean_np[t], logstd)).max()))
            assert _bits_equal(_np(tk['scaled']), sample_ref.scaled(act)), f'update {u} tick {t}: scaled action'
        check(f'update {u} stored actions = sample_ref draws (error / bound)', wa, 1.0)
        check(f'update {u} stored log-probabilities (error / bound)', wl, 1.0)
        # last_v: the value of the replayed state after the horizon
        gt = rec.gtd[u]
        sH = np.concatenate([o.state()[0] for o in oc])
        gH = np.concatenate([o.state()[1] for o in oc])
        lv64, _, _ = _forward64(P, torch.from_numpy(sH).cuda(), torch.from_numpy(gH).cuda())
        check(f'update {u} last_v', maxabs(torch.from_numpy(gt['last_value']).cuda().double() - lv64),
              2e-5 * max(1.0, maxabs(lv64)))
        # ---- c. the update, on the device's rewards checked in a
        assert _bits_equal(gt['rewards'], rewards), f'update {u}: GAE rewards'
        assert _bits_equal(gt['values'], snap['values']), f'update {u}: GAE values'
        assert np.array_equal(gt['dones'] != 0, dones), f'update {u}: GAE dones are not flag 0 (done)'
        # the C ABI takes gamma and lambda as float32 (test_gae_vs_float64_recurrence)
        tg64, adv64 = ref.gae(rewards, snap['values'], gt['last_value'], dones, float(np.float32(gt['gamma'])),
                              float(np.float32(gt['lam'])))
        for name, got, want in (('targets', gt['targets'], tg64), ('advantages', gt['advs'], adv64)):
            ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
            check(f'update {u} GAE {name} (ulps)', float((np.abs(got - want) / ulp).max()), 1.0)
        # the filter: stage 2's get_filter_index, and every row t N + i of a masked column i (stage 1: those alone)
        fd = ref.filter_index(dones) if stage == 2 else []
        masked = [t * N + i for t in range(H) for i in np.flatnonzero(col_mask)]
        fi = sorted(set(fd) | set(masked)) if masked else fd
        assert up['filter_index'] == fi, f'update {u}: filter_index'
        ev['filtered'] += len(fi)
        starts = {o.c.a for o in oc if o.c.a > 0}
        ev['boundary_runs'] += sum(1 for j in fd if j < N and j in starts)
        ev['masked_boundary_rows'] += _masked_rows_across_boundaries(fd, starts, col_mask, H, N)
        keep = ref.kept_rows(H * N, fi)
        gen = torch.Generator(device='cuda')
        gen.set_state(up['gen_state'])
        batches = []
        for _ in range(2):
            perm = torch.randperm(len(keep), device='cuda', generator=gen).cpu().numpy()
            batches += ref.minibatches(keep[perm], c['batch'], drop_last=stage == 2)
        assert len(batches) == len(up['steps']) == len(up['rows']), (len(batches), len(up['steps']), len(up['rows']))
        if stage == 1:
            assert len(batches[-1]) < c['batch'] or len(keep) % c['batch'] == 0
            ev['ragged_last'] += int(len(batches[-1]) < c['batch'])
        # the restated normalisation of the device's GAE output: over all H N rows, before np.delete (model/ppo.py:148,
        # 202, 212-218); the device forms it in float32 from float64 moments, a few u of each value (ADV_U below)
        adv_n = torch.from_numpy(ref.normalise(gt['advs'].astype(np.float64)).reshape(-1)).cuda()
        tgt_all = torch.from_numpy(gt['targets'].reshape(-1).astype(np.float64)).cuda()
        act_all = torch.from_numpy(snap['actions'].reshape(-1, 2)).cuda().double()
        lp_all = torch.from_numpy(snap['logprobs'].reshape(-1)).cuda().double()
        for k, (idx, st) in enumerate(zip(batches, up['steps'])):
            what = f'update {u} step {k} (nb {len(idx)})'
            assert st['grad_scale'] == 1.0 and st['t'] == up['step_count'] + k + 1, what
            assert _bits_equal(_np(st['p']), _np(up['flat'] if k == 0 else up['steps'][k - 1]['p1'])), \
                f'{what}: the parameters the step starts from'
            ev['steps'] += 1
            ev['steps_on_believed_gs'] += int(believed.reshape(-1)[idx].any())
            step_checks(check, what, policy, st, up['rows'][k], torch.from_numpy(idx).cuda(), x, gsx, act_all,
                        lp_all, adv_n, tgt_all, ev)
        # ---- d. the episode log lines of this update, in the trainer's (tick, column) order
        upd_lines.sort(key=lambda x: (x[0], x[1]))
        expected_lines += upd_lines
        # ---- d. the update's stats against the replay's eplog rows of ended episodes, in (tick, column) order
        ended_rows.sort(key=lambda x: (x[0], x[1]))
        ep = np.array([x[2] for x in ended_rows], np.float32).reshape(-1, 8)
        cols = np.array([x[1] for x in ended_rows], np.int64)
        s = rec.stats[u]
        want = _episode_stats(ep)
        for key in ('episodes', 'success_rate', 'mean_ep_reward'):
            assert _same(s[key], want[key]), f'update {u}: stats {key} {s[key]} != {want[key]}'
        want = {o.c.name: _episode_stats(ep[col_comp[cols] == k]) for k, o in enumerate(oc)}
        assert _same(s['by_scenario'], want), f'update {u}: by_scenario {s["by_scenario"]} != {want}'
        if pt['masked'] is None:
            assert 'by_role' not in s
        else:
            m = col_mask[cols]
            want = {'cooperative': _episode_stats(ep[~m]), pt['masked'][0]: _episode_stats(ep[m])}
            assert _same(s['by_role'], want), f'update {u}: by_role {s["by_role"]} != {want}'
            ev['episodes_cooperative'] += int((~m).sum())
            ev['episodes_masked'] += int(m.sum())
        # the planner's status shares over the update's robot-ticks (update 0's with the start's rows), in the replay's
        # statuses
        if pt['planner'] is None:
            assert 'planner' not in s
        else:
            tot = sum(o.plan.count for o in oc)
            n = int(tot.sum())
            want = {k: int(v) / n for k, v in zip(('goal_visible', 'waypoint', 'no_plan'), tot)}
            want['robot_ticks'] = n
            assert n == (H + (u == 0)) * N and _same(s['planner'], want), \
                f'update {u}: planner {s["planner"]} != {want}'
            for o in oc:
                o.plan.count[:] = 0
    # ---- d. log lines against the bookkeeping
    from rl_collision_avoidance_b200.stage_world import RESULT_STRINGS
    env_lines = [l for l in lines if isinstance(l, str) and l.startswith('Env ')]
    assert len(env_lines) == len(expected_lines) == len(cal), (len(env_lines), len(expected_lines), len(cal))
    mixed = len(oc) > 1
    for line, calv, (t, col, o, i, epi, steps, rsum, tol, goal, init, res) in zip(env_lines, cal, expected_lines):
        robot = i % o.c.env.num_env
        head = 'Env %02d, Goal (%05.1f, %05.1f), Episode %05d, setp %03d, Reward ' % (
            robot, goal[0], goal[1], epi + 1 if stage == 1 else epi, steps + 1 if stage == 1 else steps)
        assert line.startswith(head), (line, head)
        rest = line[len(head):].split(', ')
        got_r = float(rest[0])
        if stage == 1:
            dist = float(np.hypot(np.float32(goal[0]) - np.float32(init[0]), np.float32(goal[1]) - np.float32(init[1])))
            assert rest[1:] == ['Distance %05.1f' % dist, RESULT_STRINGS[res]], line
        elif mixed:
            assert rest[1:] == [RESULT_STRINGS[res], o.c.name], line
        else:
            assert rest[1:] == [RESULT_STRINGS[res] + ','], line
        # the float32 return against the float64 sum of the rewards PPO trained on, within OracleComponent.tick's bound
        assert abs(float(calv) - rsum) <= tol + 1e-30, (line, float(calv), rsum, tol)
        assert abs(got_r - rsum) <= 0.05 + tol + 1e-9, (line, rsum)
    check.done()
    # ---- the events each case exists for
    print(f'[events] {case}: {dict(ev)}, train {t_train:.1f} s, total {time.perf_counter() - t_start:.1f} s')
    assert ev['ended'] > 0 and len(env_lines) > 0 and ev['steps'] > 0
    if case in ('stage1', 'noise', 'latency', 'planner_stage1'):
        assert ev['ended_last_tick'] > 0 and ev['respawn'] > 0
    if noise is not None:
        assert ev['noised_rows'] > 0
    if case in ('stage2', 'mix', 'dynamics'):
        assert ev['filtered'] > 0 and ev['idle'] > 0 and ev['respawn'] > 0
    if case in ('random', 'mix', 'localization', 'planner_straight'):
        assert ev['relaid'] > 0
    if case in ('arena', 'planner_chain'):
        assert ev['relaid'] > 0 and ev['idle'] > 0 and ev['filtered'] > 0
    if case == 'mix':
        assert ev['boundary_runs'] > 0, 'no filter run crossed a component boundary'
    if case == 'latency':
        assert ev['scan_delayed'] > 0 and ev['command_delayed'] > 0, 'no delayed scan or command'
        assert ev['ring_restart_on_boundary'] > 0, 'no command ring restarted on the horizon boundary'
    if case == 'dynamics':
        assert ev['clamped'] > 0, 'no limit was reached'
        assert ev['crash_prev_reset'] > 0, 'no moving robot crashed'
    if case == 'localization':
        assert ev['believed'] > 0 and ev['relaid_sigma_redrawn'] > 0, 'no believed gs or no redrawn sigma'
        assert ev['steps_on_believed_gs'] == ev['steps'], 'a PPO step on true gs alone'
    if case == 'masked_stage1':
        assert ev['masked_checked'] > 0 and ev['masked_changed'] > 0 and ev['filtered'] > 0
        assert ev['ragged_last'] == 2, 'the kept rows filled the last minibatch'
        assert ev['episodes_cooperative'] > 0 and ev['episodes_masked'] > 0, 'a role without episodes'
    if case == 'chain':
        for link in ('masked_changed', 'command_delayed', 'noised_rows', 'limited', 'scan_delayed', 'noised_scans',
                     'believed'):
            assert ev[link] > 0, f'{link}: this link changed no row'
        assert ev['masked_checked'] > 0 and ev['episodes_masked'] > 0
        assert ev['masked_boundary_rows'] > 0, 'no masked row in a filter run crossing a component boundary'
    if pt['planner'] is not None:
        assert ev['replanned'] > 0 and ev['status_0'] > 0 and ev['status_1'] > 0, 'no re-plan, or a status unseen'
        assert ev['exempt'] <= max(1, ev['plan_rows'] // 1000), 'too many rows whose waypoint the walks disagree on'
    if pt['planner'] == 'geodesic':
        assert ev['shaped_changed'] > 0, 'no shaped reward differed from the tick\'s'
        assert ev['corrected'] > 0, 'no ended episode had its return corrected'
        assert ev['straddled'] > 0, 'no episode straddled the update boundary'
    if case == 'planner_chain':
        for link in ('masked_changed', 'command_delayed', 'noised_rows', 'limited', 'scan_delayed', 'noised_scans'):
            assert ev[link] > 0, f'{link}: this link changed no row'
        assert ev['masked_checked'] > 0 and ev['episodes_masked'] > 0
