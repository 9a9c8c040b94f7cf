"""Shared rollout/update loop of the stage-1 / stage-2 trainers (the body of `run()` in
/root/reference/ppo_stage1.py:39-131 and ppo_stage2.py:39-138, batched on the device).

One process per GPU.  Per tick: policy forward + sampling (librlca.so) -> fused env tick (librlca.so) with
every output written straight into the rollout buffers; every HORIZON ticks: GAE, PPO update with an NCCL
all-reduce of the flat gradient per optimizer step when launched under torchrun.  No mpi4py, no ROS.
A stage-2 run may tick several env handles, one per scenario, on column slices of one rollout (DESIGN.md §9l).
"""
from __future__ import annotations

import os
import time

import numpy as np
import torch

from .mix import MIX_AUTO_RESET, MIX_SCENARIOS, SLICE_ALIGN, check_aligned
from .model.ppo import generate_action, generate_train_data, ppo_update_stage1, ppo_update_stage2
from .model.utils import get_filter_index
from .crowd import Crowd
from .dynamics import Dynamics
from .evaluation import non_cooperative_mask
from .latency import Latency
from .localization import Localization
from .noise import Noise
from .orca import NonCooperative
from .planner import Planner
from .stage_world import RESULT_STRINGS


def _episode_stats(ep):
    """Episodes, success and crash rates and mean episode reward of eplog rows (E, 8)."""
    n = len(ep)
    nan = float('nan')
    return {'episodes': n, 'success_rate': float((ep[:, 6] == 1).mean()) if n else nan,
            'crash_rate': float((ep[:, 6] == 2).mean()) if n else nan,
            'mean_ep_reward': float(ep[:, 2].mean()) if n else nan}


class Rollout:
    """Device-resident rollout storage: the reference's `buff` list (ppo_stage1.py:102-103) as tensors."""

    def __init__(self, horizon, n, beams, device):
        self.stacks = torch.empty(horizon + 1, n, 3, beams, device=device)   # scan FIFOs, slot t+1 written by tick t
        self.gs = torch.empty(horizon + 1, n, 4, device=device)             # local goal + speed
        self.actions = torch.empty(horizon, n, 2, device=device)
        self.scaled = torch.empty(n, 2, device=device)
        self.logprobs = torch.empty(horizon, n, device=device)
        self.values = torch.empty(horizon, n, device=device)
        self.rewards = torch.empty(horizon, n, device=device)
        self.flags = torch.zeros(horizon, n, 4, dtype=torch.uint8, device=device)
        self.eplog = torch.zeros(horizon, n, 8, device=device)


class _Component:
    """One env handle of a run and its views of the rollout: agent columns [a, b), sliced once."""

    def __init__(self, env, ro, a, b, noise=None, latency=None, dynamics=None, localization=None):
        self.env, self.a, self.b = env, a, b
        self.noise = noise                              # noise.Noise of the env, or None
        self.latency = latency                          # latency.Latency of the env, or None
        self.dynamics = dynamics                        # dynamics.Dynamics of the env, or None
        self.localization = localization                # localization.Localization of the env, or None
        self.masked = None                              # orca.NonCooperative or crowd.Crowd of the env, or None
        self.planner = None                             # planner.Planner of the env (steering), or None
        self.ticked = False                             # a tick has run, so self.flags holds its flags
        self.name = env.sc.name
        self.relayout = env.sc.layout is not None
        self.scaled = ro.scaled[a:b]
        self.stacks = ro.stacks[:, a:b]
        self.gs = ro.gs[:, a:b]
        self.rewards = ro.rewards[:, a:b]
        self.flags = ro.flags[:, a:b]
        self.eplog = ro.eplog[:, a:b]

    def check_aligned(self):
        for name, view in (('action', self.scaled), ('stack', self.stacks), ('gs', self.gs),
                           ('reward', self.rewards), ('flags', self.flags), ('eplog', self.eplog)):
            check_aligned('%s[%d:%d] of %s' % (name, self.a, self.b, self.name), view, SLICE_ALIGN[name])

    def start(self):
        """The env's first episode, and slot 0 of its stacks and gs."""
        e = self.env
        e.reset_world()                                 # ppo_stage1.py:46-47
        e.reset_pose()                                  # :50
        e.generate_goal_point()                         # :52
        if self.relayout:
            e.random_layout()                           # the first layout, as evaluate() draws it
        obs = e.get_laser_observation()
        self.stacks[0] = obs[:, None, :]                # deque([obs, obs, obs]) (:60)
        if self.latency is not None:
            self.latency.scan(self.stacks[0])           # every row starts an episode: its rings hold the first scan
        if self.noise is not None:
            self.noise.scan(self.stacks[0])             # what a noisy robot's first scan reads, in all three slots
        self.gs[0] = e.gs
        if self.localization is not None:
            self.localization.observe(gs=self.gs[0], out=self.gs[0])    # every row starts an episode
        if self.planner is not None:
            self.planner.update(None, gs=self.gs[0])    # the first waypoints; every row starts an episode

    def tick(self, t):
        """Tick t on the component's slices, after the policy has written ro.scaled.  With noise the robots execute
        noise.action's command (ro.scaled, which PPO's actions were drawn with, is not written) and the stack the tick
        and the re-layout wrote is perturbed as a noisy robot would read it.  With latency the command is delayed
        first, with the flags of the tick before (at t = 0 slot H - 1 of the previous rollout, still intact; None on
        the run's first tick), and the stack is delayed after the re-layout and before any noise.  With dynamics the
        command, last of all, is limited in acceleration, with the same flags of the tick before.  With localization
        the gs the tick and the re-layout wrote becomes, in place and last of all, the gs the robot believes, with the
        flags of this tick.  With masked agents their rows of ro.scaled are overwritten first, before any latency; PPO
        keeps the policy's sampled action in ro.actions.  With a planner the gs the tick and the re-layout wrote becomes,
        in place and last of all, the waypoint gs, and a reward planner shapes the tick's reward and the returns of the
        episodes it ended in place, with the flags as the re-layout left them."""
        e = self.env
        if self.masked is not None:
            self.masked.apply(self.scaled)
        cmd = self.scaled
        prev = self.flags[t - 1] if t > 0 else self.flags[-1] if self.ticked else None
        if self.latency is not None:
            cmd = self.latency.action(cmd, prev)
        self.ticked = True
        if self.noise is not None:
            cmd = self.noise.action(cmd)
        if self.dynamics is not None:
            cmd = self.dynamics.action(cmd, prev)
        e.control_vel(cmd, live=e.live if self.relayout else None, stack_in=self.stacks[t],
                      stack_out=self.stacks[t + 1],
                      out={'reward': self.rewards[t], 'flags': self.flags[t], 'gs': self.gs[t + 1],
                           'eplog': self.eplog[t]})
        if self.relayout:
            e.relayout_finished(self.stacks[t + 1], out={'gs': self.gs[t + 1], 'flags': self.flags[t]})
        if self.latency is not None:
            self.latency.scan(self.stacks[t + 1], self.flags[t])
        if self.noise is not None:
            self.noise.scan(self.stacks[t + 1], self.flags[t])
        if self.localization is not None:
            self.localization.observe(self.flags[t], gs=self.gs[t + 1], out=self.gs[t + 1])
        if self.planner is not None:
            self.planner.update(self.flags[t], reward=self.rewards[t], eplog=self.eplog[t], gs=self.gs[t + 1])


def compose(envs, ro, noise=None, latency=None, dynamics=None, localization=None):
    """The components of `envs` on the rollout `ro`: env k owns the agent columns that follow env k - 1's.  With more
    than one env, ValueError for a slice the kernels cannot read at its alignment (mix.SLICE_ALIGN).  `noise`
    (noise.NoiseParams) gives component k a noise.Noise with stream id k, `latency` (latency.LatencyParams) a
    latency.Latency with stream id k, `dynamics` (dynamics.DynamicsParams) a dynamics.Dynamics with stream id k and
    `localization` (localization.LocalizationParams) a localization.Localization with stream id k."""
    comps, a = [], 0
    for k, e in enumerate(envs):
        comps.append(_Component(e, ro, a, a + e.N, None if noise is None else Noise(e, noise, stream_id=k),
                                None if latency is None else Latency(e, latency, stream_id=k),
                                None if dynamics is None else Dynamics(e, dynamics, stream_id=k),
                                None if localization is None else Localization(e, localization, stream_id=k)))
        a += e.N
    if a != ro.scaled.shape[0]:
        raise ValueError('the envs hold %d agents, the rollout %d' % (a, ro.scaled.shape[0]))
    if len(comps) > 1:
        for c in comps:
            c.check_aligned()
    return comps


PLANNERS = ('geodesic', 'straight')


def attach_planners(comps, planner, localization=None, tables=None):
    """Give every component a planner.Planner of its env that steers by waypoints: 'geodesic' also shapes the reward by
    geodesic progress, 'straight' keeps the tick's reward.  None attaches nothing.  `tables`: one
    planner.PlannerTables per component (build_plan_tables of its env's map), or None to build them here.  ValueError
    for another value, with localization error (the planner plans from the true pose) and, naming the map and the
    limit, for a map the planner refuses (build_plan_tables)."""
    if planner is None:
        return
    if planner not in PLANNERS:
        raise ValueError('planner must be None or one of %s, got %r' % (', '.join(PLANNERS), planner))
    if localization is not None:
        raise ValueError('the planner plans from the true pose; localization error needs a planner on the believed '
                         'pose')
    if tables is not None and len(tables) != len(comps):
        raise ValueError('planner tables: %d given for %d components' % (len(tables), len(comps)))
    for k, c in enumerate(comps):
        c.planner = Planner(c.env, steer=True, reward=planner == 'geodesic',
                            tables=None if tables is None else tables[k])


def _status_shares(comps):
    """The share of robot-ticks of each planner status since the last call, over every component's rows; zeroes the
    counts."""
    tot = sum(c.planner.status_count.to(torch.int64).sum(0) for c in comps).cpu().numpy()
    for c in comps:
        c.planner.status_count.zero_()
    n = int(tot.sum())
    out = {k: (int(v) / n if n else float('nan')) for k, v in zip(('goal_visible', 'waypoint', 'no_plan'), tot)}
    out['robot_ticks'] = n
    return out


def masked_agents(comps, non_cooperative=None, crowd=None):
    """Give every component its masked agents and return the (N,) bool mask of the rollout's masked columns, or None
    when there are none.  non_cooperative = (k, speed or None): an orca.NonCooperative; crowd = (k, crowd.CrowdParams,
    map flag): a crowd.Crowd (DESIGN.md §9t); in both, robots floor(j R_c / k), j < k, of every world of component c
    (evaluation.non_cooperative_mask: ValueError unless 1 <= k <= R_c).  ValueError for both."""
    if non_cooperative is not None and crowd is not None:
        raise ValueError('crowd and non_cooperative cannot be combined: the stats split into two roles')
    if non_cooperative is None and crowd is None:
        return None
    k = non_cooperative[0] if non_cooperative is not None else crowd[0]
    masks = [non_cooperative_mask(c.env.cfg.robots_per_world, c.env.cfg.num_worlds, k) for c in comps]
    for c, m in zip(comps, masks):
        if non_cooperative is not None:
            c.masked = NonCooperative(c.env, m, speed=non_cooperative[1])
        else:
            c.masked = Crowd(c.env, m, crowd[1], obstacles=crowd[2])
    return np.concatenate(masks) != 0


def masked_rows(H, col_mask):
    """Every row t * N + i of a masked column i, sorted: stage 1's filter."""
    N = col_mask.shape[0]
    return (np.arange(H)[:, None] * N + np.flatnonzero(col_mask)[None, :]).reshape(-1).tolist()


def masked_filter_index(dones, col_mask):
    """Stage 2's filter with masked columns: get_filter_index(dones) over every column (the reference's quirk
    unchanged) united with masked_rows, sorted."""
    return np.union1d(np.asarray(get_filter_index(dones), np.int64), masked_rows(dones.shape[0], col_mask)).tolist()


def _check_mix(envs, stage):
    """ValueError unless `envs` can share one stage-2 rollout (DESIGN.md §9l)."""
    if stage != 2:
        raise ValueError('a mix of scenarios trains with stage 2, got stage %d' % stage)
    seen = set()
    for e in envs:
        name, ar = e.sc.name, int(e.cfg.auto_reset)
        if name == 'stage1':
            raise ValueError("stage 1 cannot be mixed: it re-spawns each robot on its own and trains with stage 1's "
                             'update')
        if name not in MIX_SCENARIOS:
            raise ValueError('scenario %r cannot be mixed (one of %s)' % (name, ', '.join(MIX_SCENARIOS)))
        if name in seen:
            raise ValueError('scenario %s appears more than once in the mix' % name)
        seen.add(name)
        if ar != MIX_AUTO_RESET[name]:
            raise ValueError('%s trains with auto_reset %d in a mix, got %d' % (name, MIX_AUTO_RESET[name], ar))
        if e.device != envs[0].device or e.beam_mum != envs[0].beam_mum:
            raise ValueError('the envs of a mix must share the device and the beam count: %s has %s / %d, %s has %s / %d'
                             % (envs[0].sc.name, envs[0].device, envs[0].beam_mum, name, e.device, e.beam_mum))


def run(env, policy, policy_path, action_bound, optimizer, hp, logger=None, logger_cal=None, stage=1, max_updates=None,
        process_group=None, rank=0, save_every=20, generator=None, start_update=0, diagnostics=False, target_kl=None,
        noise=None, latency=None, dynamics=None, localization=None, non_cooperative=None, crowd=None, planner=None,
        planner_tables=None):
    """hp: dict with HORIZON, GAMMA, LAMDA, BATCH_SIZE, EPOCH, COEFF_ENTROPY, CLIP_VALUE, NUM_ENV, OBS_SIZE, ACT_SIZE,
    LASER_HIST, MAX_EPISODES.  `start_update` continues the checkpoint numbering of a resumed run.
    A random scenario (env.sc.layout, DESIGN.md §9k) trains with stage 2's update on per-world layouts: the env runs
    with auto_reset 0, every tick passes env.live and is followed by env.relayout_finished, and a world whose robots
    have all ended their episodes gets a new layout.
    `env` may be a sequence of envs, one per scenario (DESIGN.md §9l): stage 2 and the circle with auto_reset 2 and a
    random scenario with auto_reset 0, each at most once, with stage 2.  Component k owns the rollout's agent columns
    [a_k, b_k) in the order given; every tick runs one policy forward over all N = sum N_k columns, then each
    component's tick (and re-layout) on its slices, and each update is stage 2's over the whole (H, N) batch.  A
    one-element sequence is the single-env run.
    `diagnostics` (DESIGN.md §9n) adds stats[k]['diagnostics'], the metrics of model.diagnostics.metrics plus
    'epochs_run' and 'logstd', and rank 0 writes one line per update to the diag.log logger; `target_kl` (finite and
    > 0, implies diagnostics) skips the remaining epochs of an update once an epoch's approx_kl_k3 exceeds it.
    `noise` (noise.NoiseParams, DESIGN.md §9p) trains under sensor and actuation noise: component k gets a noise.Noise
    with stream id k, its robots execute the perturbed command and every stack the policy reads is perturbed; the
    env's world_offset makes the draws of each data-parallel rank differ.  None issues no noise launch.
    `latency` (latency.LatencyParams, DESIGN.md §9q) trains under sensing and command latency: component k gets a
    latency.Latency with stream id k, its robots execute the command of l ticks earlier and read the scan of d ticks
    earlier, both before any noise; PPO still stores the issued action and its log-probability.  None launches nothing.
    `dynamics` (dynamics.DynamicsParams, DESIGN.md §9r) trains under acceleration limits: component k gets a
    dynamics.Dynamics with stream id k, applied to the command last, after any noise; PPO still stores the issued
    action.  None launches nothing.
    `localization` (localization.LocalizationParams, DESIGN.md §9s) trains under localization error: component k gets
    a localization.Localization with stream id k, and every gs the policy reads (ro.gs, slot 0 and every slot a tick
    wrote, after any re-layout) is the believed one, so PPO stores and re-evaluates what the policy read.  Rewards and
    episode ends stay on the true state.  None launches nothing.
    `non_cooperative` ((k, speed or None), DESIGN.md §9h) or `crowd` ((k, crowd.CrowdParams, map flag), §9t) puts k
    masked agents into every world of every component (masked_agents); their rows of the action are overwritten before
    any latency, and every row of their columns is left out of every PPO update (stage 1: filter_index; stage 2:
    united with get_filter_index).  The stats then also hold 'by_role' {'cooperative', 'non_cooperative' or 'crowd'}.
    `planner` ('geodesic' or 'straight', DESIGN.md §9x) gives component k a planner.Planner (attach_planners): every
    gs the policy reads (ro.gs, slot 0 and every slot a tick wrote, after any re-layout) is the waypoint gs, so PPO
    stores and re-evaluates what the policy read; 'geodesic' also shapes ro.rewards and the episodes' returns by
    geodesic progress, 'straight' keeps the tick's reward.  The stats then also hold 'planner', the status shares of the
    update's robot-ticks.  Refused with localization error and on maps the planner refuses.  None launches nothing.
    `planner_tables` (one planner.PlannerTables per env, in order) saves building the planning graphs again.
    Returns per-update stats (for tests / benchmarks); 'by_scenario' splits the episodes by component."""
    envs = list(env) if isinstance(env, (list, tuple)) else [env]
    if not envs:
        raise ValueError('trainer.run needs at least one env')
    mixed = len(envs) > 1
    for e in envs:
        if e.sc.layout is not None and (stage != 2 or int(e.cfg.auto_reset) != 0):
            raise ValueError('a random scenario trains with stage 2 and auto_reset 0 (per-world re-layouts), got stage '
                             '%d and auto_reset %d' % (stage, int(e.cfg.auto_reset)))
    if mixed:
        _check_mix(envs, stage)
    H, N = hp['HORIZON'], sum(e.N for e in envs)
    dev = envs[0].device
    ro = Rollout(H, N, envs[0].beam_mum, dev)
    comps = compose(envs, ro, noise, latency, dynamics, localization)
    attach_planners(comps, planner, localization, planner_tables)
    col_mask = masked_agents(comps, non_cooperative, crowd)
    role = 'crowd' if crowd is not None else 'non_cooperative'
    col_comp = np.repeat(np.arange(len(comps)), [e.N for e in envs])     # component of every agent column
    for c in comps:
        c.start()
    diag = None
    if diagnostics or target_kl is not None:
        from .model.diagnostics import PPODiagnostics, check_target_kl, format_line, logger_diag
        if target_kl is not None:
            target_kl = check_target_kl(target_kl)
        diag = PPODiagnostics(policy, hp['EPOCH'], action_bound)
    global_update = int(start_update)
    updates_done = 0
    episodes = 0
    stats = []
    while True:
        t0 = time.perf_counter()
        for t in range(H):
            generate_action(env=envs[0], state_list=(ro.stacks[t], ro.gs[t]), policy=policy, action_bound=action_bound,
                            out={'value': ro.values[t], 'action': ro.actions[t], 'logprob': ro.logprobs[t],
                                 'scaled': ro.scaled})
            for c in comps:
                c.tick(t)
        # last_v from the state after the horizon (ppo_stage1.py:94-97)
        last_v, _ = policy.forward_values(ro.stacks[H], ro.gs[H])
        dones = ro.flags[:, :, 0]
        t_batch, advs_batch = generate_train_data(rewards=ro.rewards, gamma=hp['GAMMA'], values=ro.values,
                                                  last_value=last_v, dones=dones, lam=hp['LAMDA'])
        torch.cuda.synchronize(dev)
        t1 = time.perf_counter()
        for c in comps:
            if c.relayout:
                c.env.check_relayout()
        memory = (ro.stacks[:H], ro.gs[:H, :, 0:2], ro.gs[:H, :, 2:4], ro.actions, ro.logprobs, t_batch, ro.values,
                  ro.rewards, advs_batch)
        common = dict(policy=policy, optimizer=optimizer, batch_size=hp['BATCH_SIZE'], memory=memory, epoch=hp['EPOCH'],
                      coeff_entropy=hp['COEFF_ENTROPY'], clip_value=hp['CLIP_VALUE'], num_step=H, num_env=N,
                      frames=hp['LASER_HIST'], obs_size=hp['OBS_SIZE'], act_size=hp['ACT_SIZE'], generator=generator,
                      process_group=process_group, diagnostics=diag, target_kl=target_kl)
        if stage == 1:
            if col_mask is None:
                rows = ppo_update_stage1(**common)
            else:
                rows = ppo_update_stage1(filter_index=masked_rows(H, col_mask), **common)
        else:
            # ppo_stage2.py:112.  The reference's run counter is not reset between columns, so a run of done carries
            # from one robot's column into the next; in a mix it carries across the boundary between two components
            # in the same way (§9l), exactly as for one env of N columns.
            filter_index = get_filter_index(dones) if col_mask is None else masked_filter_index(dones, col_mask)
            rows = ppo_update_stage2(filter_index=filter_index, **common)
        torch.cuda.synchronize(dev)
        t2 = time.perf_counter()
        global_update += 1
        updates_done += 1
        # ---- episode log lines (ppo_stage1.py:127-131 / ppo_stage2.py:136-137), one D2H per update
        fl = ro.flags.cpu().numpy()
        ended = (fl[:, :, 0] != 0) & (fl[:, :, 2] != 0) if stage == 2 else (fl[:, :, 0] != 0)
        ep = ro.eplog.cpu().numpy()[ended]
        idx = np.argwhere(ended)
        for (tt, i), e in zip(idx, ep):
            episodes += 1
            if logger is not None and rank == 0:
                res = RESULT_STRINGS.get(int(e[6]), 0)
                c = comps[col_comp[i]]
                robot = (i - c.a) % c.env.num_env           # the robot's index within its own component's world
                if stage == 1:
                    dist = float(np.hypot(e[0] - e[4], e[1] - e[5]))
                    logger.info('Env %02d, Goal (%05.1f, %05.1f), Episode %05d, setp %03d, Reward %-5.1f, Distance %05.1f, %s' %
                                (robot, e[0], e[1], int(e[7]), int(e[3]) + 1, e[2], dist, res))
                elif mixed:
                    logger.info('Env %02d, Goal (%05.1f, %05.1f), Episode %05d, setp %03d, Reward %-5.1f, %s, %s' %
                                (robot, e[0], e[1], int(e[7]) - 1, int(e[3]), e[2], res, c.name))
                else:
                    logger.info('Env %02d, Goal (%05.1f, %05.1f), Episode %05d, setp %03d, Reward %-5.1f, %s,' %
                                (robot, e[0], e[1], int(e[7]) - 1, int(e[3]), e[2], res))
            if logger_cal is not None and rank == 0:
                logger_cal.info(float(e[2]))
        if rank == 0 and policy_path and global_update % save_every == 0:
            name = '/Stage1_{}'.format(global_update) if stage == 1 else '/stage2_{}.pth'.format(global_update)
            torch.save(policy.state_dict(), policy_path + name)                      # ppo_stage1.py:122-126
            torch.save({'optimizer': optimizer.state_dict(), 'update': global_update,
                        'sample_counter': policy.sample_counter}, policy_path + name + '.trainer')
            if logger is not None:
                logger.info('########################## model saved when update {} times#########'
                            '################'.format(global_update))
        ep_comp = col_comp[idx[:, 1]]
        stats.append({'update': global_update, 'rollout_s': t1 - t0, 'update_s': t2 - t1,
                      'agent_steps_per_s': H * N / (t2 - t0), 'episodes': len(ep),
                      'mean_ep_reward': float(ep[:, 2].mean()) if len(ep) else float('nan'),
                      'success_rate': float((ep[:, 6] == 1).mean()) if len(ep) else float('nan'),
                      'losses': rows[-1] if rows else None,
                      'by_scenario': {c.name: _episode_stats(ep[ep_comp == k]) for k, c in enumerate(comps)}})
        if col_mask is not None:
            ep_masked = col_mask[idx[:, 1]]
            stats[-1]['by_role'] = {'cooperative': _episode_stats(ep[~ep_masked]), role: _episode_stats(ep[ep_masked])}
        if planner is not None:
            stats[-1]['planner'] = _status_shares(comps)
        if diag is not None:
            stats[-1]['diagnostics'] = diag.metrics()
            if rank == 0:
                logger_diag.info(format_line(global_update, stats[-1]['diagnostics']))
        # carry the state over the horizon boundary
        ro.stacks[0].copy_(ro.stacks[H])
        ro.gs[0].copy_(ro.gs[H])
        stop = (max_updates is not None and updates_done >= max_updates) or episodes >= hp['MAX_EPISODES'] * N
        if process_group is not None:
            # episode counts are rank-local: leave together, or the others hang in the next all-reduce
            from .parallel import agree_to_stop
            stop = agree_to_stop(stop, dev, None if process_group is True else process_group)
        if stop:
            break
    return stats
