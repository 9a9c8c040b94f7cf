"""Shared rollout/update loop of the stage-1 / stage-2 trainers (the body of `run()` in
/root/reference/ppo_stage1.py:39-131 and ppo_stage2.py:39-138, batched on the device).

One process per GPU.  Per tick: policy forward + sampling (librlca.so) -> fused env tick (librlca.so) with
every output written straight into the rollout buffers; every HORIZON ticks: GAE, PPO update with an NCCL
all-reduce of the flat gradient per optimizer step when launched under torchrun.  No mpi4py, no ROS.
"""
from __future__ import annotations

import os
import time

import numpy as np
import torch

from .model.ppo import generate_action, generate_train_data, ppo_update_stage1, ppo_update_stage2
from .model.utils import get_filter_index
from .stage_world import RESULT_STRINGS


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


def run(env, policy, policy_path, action_bound, optimizer, hp, logger=None, logger_cal=None, stage=1, max_updates=None,
        process_group=None, rank=0, save_every=20, generator=None, start_update=0):
    """hp: dict with HORIZON, GAMMA, LAMDA, BATCH_SIZE, EPOCH, COEFF_ENTROPY, CLIP_VALUE, NUM_ENV, OBS_SIZE, ACT_SIZE,
    LASER_HIST, MAX_EPISODES.  `start_update` continues the checkpoint numbering of a resumed run.
    A random scenario (env.sc.layout, DESIGN.md §9k) trains with stage 2's update on per-world layouts: the env runs
    with auto_reset 0, every tick passes env.live and is followed by env.relayout_finished, and a world whose robots
    have all ended their episodes gets a new layout.
    Returns per-update stats (for tests / benchmarks)."""
    relayout = env.sc.layout is not None
    if relayout and (stage != 2 or int(env.cfg.auto_reset) != 0):
        raise ValueError('a random scenario trains with stage 2 and auto_reset 0 (per-world re-layouts), got stage %d '
                         'and auto_reset %d' % (stage, int(env.cfg.auto_reset)))
    H, N = hp['HORIZON'], env.N
    dev = env.device
    ro = Rollout(H, N, env.beam_mum, dev)
    env.reset_world()                                   # ppo_stage1.py:46-47
    env.reset_pose()                                    # :50
    env.generate_goal_point()                           # :52
    if relayout:
        env.random_layout()                             # the first layout, as evaluate() draws it
    obs = env.get_laser_observation()
    ro.stacks[0] = obs[:, None, :]                      # deque([obs, obs, obs]) (:60)
    ro.gs[0] = env.gs
    global_update = int(start_update)
    updates_done = 0
    episodes = 0
    stats = []
    while True:
        t0 = time.perf_counter()
        for t in range(H):
            generate_action(env=env, state_list=(ro.stacks[t], ro.gs[t]), policy=policy, action_bound=action_bound,
                            out={'value': ro.values[t], 'action': ro.actions[t], 'logprob': ro.logprobs[t],
                                 'scaled': ro.scaled})
            env.control_vel(ro.scaled, live=env.live if relayout else None, stack_in=ro.stacks[t],
                            stack_out=ro.stacks[t + 1],
                            out={'reward': ro.rewards[t], 'flags': ro.flags[t], 'gs': ro.gs[t + 1], 'eplog': ro.eplog[t]})
            if relayout:
                env.relayout_finished(ro.stacks[t + 1], out={'gs': ro.gs[t + 1], 'flags': ro.flags[t]})
        # last_v from the state after the horizon (ppo_stage1.py:94-97)
        last_v, _ = policy.forward_values(ro.stacks[H], ro.gs[H])
        dones = ro.flags[:, :, 0]
        t_batch, advs_batch = generate_train_data(rewards=ro.rewards, gamma=hp['GAMMA'], values=ro.values,
                                                  last_value=last_v, dones=dones, lam=hp['LAMDA'])
        torch.cuda.synchronize(dev)
        t1 = time.perf_counter()
        if relayout:
            env.check_relayout()
        memory = (ro.stacks[:H], ro.gs[:H, :, 0:2], ro.gs[:H, :, 2:4], ro.actions, ro.logprobs, t_batch, ro.values,
                  ro.rewards, advs_batch)
        common = dict(policy=policy, optimizer=optimizer, batch_size=hp['BATCH_SIZE'], memory=memory, epoch=hp['EPOCH'],
                      coeff_entropy=hp['COEFF_ENTROPY'], clip_value=hp['CLIP_VALUE'], num_step=H, num_env=N,
                      frames=hp['LASER_HIST'], obs_size=hp['OBS_SIZE'], act_size=hp['ACT_SIZE'], generator=generator,
                      process_group=process_group)
        if stage == 1:
            rows = ppo_update_stage1(**common)
        else:
            filter_index = get_filter_index(dones)            # ppo_stage2.py:112
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
                if stage == 1:
                    dist = float(np.hypot(e[0] - e[4], e[1] - e[5]))
                    logger.info('Env %02d, Goal (%05.1f, %05.1f), Episode %05d, setp %03d, Reward %-5.1f, Distance %05.1f, %s' %
                                (i % env.num_env, e[0], e[1], int(e[7]), int(e[3]) + 1, e[2], dist, res))
                else:
                    logger.info('Env %02d, Goal (%05.1f, %05.1f), Episode %05d, setp %03d, Reward %-5.1f, %s,' %
                                (i % env.num_env, e[0], e[1], int(e[7]) - 1, int(e[3]), e[2], res))
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
        stats.append({'update': global_update, 'rollout_s': t1 - t0, 'update_s': t2 - t1,
                      'agent_steps_per_s': H * N / (t2 - t0), 'episodes': len(ep),
                      'mean_ep_reward': float(ep[:, 2].mean()) if len(ep) else float('nan'),
                      'success_rate': float((ep[:, 6] == 1).mean()) if len(ep) else float('nan'),
                      'losses': rows[-1] if rows else None})
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
