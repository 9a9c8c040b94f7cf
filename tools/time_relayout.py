#!/usr/bin/env python
"""The cost numbers of DESIGN.md §9k: one StageWorld.relayout_finished call (rlca_layout_respawn, rlca_env_observe and
rlca_stack_refresh) on random K = 16 at 256 and 1024 worlds, once with no world finishing and once with every world
re-laid, and one tick of the same env (rlca_env_step with the live mask and the scan stacks), each timed twice with
CUDA events round every call; then training agent-steps/s from trainer.run's own stats, random K = 16 against stage 2
at a similar number of agents, with ppo_stage2.py's hyper-parameters.  Prints the card and power limit first.

    python tools/time_relayout.py
"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ppo_stage1  # noqa: E402
import ppo_stage2  # noqa: E402
from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario, random_max_ticks  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402
from rl_collision_avoidance_b200.trainer import run  # noqa: E402

K, CALLS = 16, 200


def _env(worlds):
    sc = make_scenario('random', robots_per_world=K, timeout=random_max_ticks(10.0))
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=0, auto_reset=0)
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    env.random_layout()
    return env


def _per_call_us(fn, before=None, calls=CALLS):
    """Mean of CUDA-event times round each of `calls` calls of fn (`before` runs outside the timed window)."""
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(calls)]
    for _ in range(10):
        if before:
            before()
        fn()
    for e0, e1 in evs:
        if before:
            before()
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return 1e3 * float(np.mean([e0.elapsed_time(e1) for e0, e1 in evs]))


def time_calls(worlds):
    env = _env(worlds)
    n = env.N
    stacks = torch.empty(2, n, 3, 512, device='cuda')
    stacks[0] = env.obs[:, None, :]
    gs = torch.empty(2, n, 4, device='cuda')
    flags = torch.zeros(n, 4, dtype=torch.uint8, device='cuda')
    out = {'gs': gs[1], 'flags': flags}
    action = torch.zeros(n, 2, device='cuda')
    relayout = lambda: env.relayout_finished(stacks[1], out=out)
    latch_all = lambda: env.state['meta'][:, 3].fill_(1)
    tick = lambda: env.control_vel(action, live=env.live, stack_in=stacks[0], stack_out=stacks[1],
                                   out={'gs': gs[1], 'flags': flags})
    rows = []
    for _ in range(2):
        quiet = _per_call_us(relayout)
        torch.cuda.synchronize()
        assert not env.state['meta'][:, 3].any()
        full = _per_call_us(relayout, before=latch_all)
        torch.cuda.synchronize()
        assert bool(flags[:, 3].all()) and not env._relayout_status.any()
        flags.zero_()
        env.state['meta'][:, 3].zero_()
        t = _per_call_us(tick, calls=CALLS)
        rows.append((quiet, full, t))
        env.state['meta'][:, 3].zero_()
        env.live.fill_(1)
    return rows


def train_rate(env, updates=4):
    policy = CNNPolicy(frames=3, action_space=2, seed=0, max_batch=max(ppo_stage2.BATCH_SIZE, env.N))
    policy.load_state_dict(torch.load(os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth'),
                                      map_location='cuda'))
    opt = Adam(policy.parameters(), lr=ppo_stage1.LEARNING_RATE)
    hp = dict(HORIZON=ppo_stage1.HORIZON, GAMMA=ppo_stage1.GAMMA, LAMDA=ppo_stage1.LAMDA,
              BATCH_SIZE=ppo_stage2.BATCH_SIZE, EPOCH=ppo_stage2.EPOCH, COEFF_ENTROPY=ppo_stage1.COEFF_ENTROPY,
              CLIP_VALUE=ppo_stage1.CLIP_VALUE, NUM_ENV=env.num_env, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3,
              MAX_EPISODES=ppo_stage1.MAX_EPISODES)
    stats = run(env=env, policy=policy, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp,
                stage=2, max_updates=updates, generator=torch.Generator(device='cuda').manual_seed(0))
    s = stats[1:]                                                # the first update warms up
    return (float(np.mean([x['agent_steps_per_s'] for x in s])), float(np.mean([x['rollout_s'] for x in s])),
            float(np.mean([x['update_s'] for x in s])))


def main():
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    for worlds in (256, 1024):
        for i, (quiet, full, tick) in enumerate(time_calls(worlds)):
            print('%d x %d agents, pass %d: relayout_finished %.1f us (no world finishing), %.1f us (every world '
                  're-laid); one tick %.1f us (mean of %d calls)' % (worlds, K, i + 1, quiet, full, tick, CALLS),
                  flush=True)
        torch.cuda.empty_cache()
    from rl_collision_avoidance_b200.stage_world2 import StageWorld as Stage2World
    for name, env in (('random K = 16, 256 worlds', _env(256)),
                      ('stage 2, 93 worlds', Stage2World(512, index=0, num_env=44, num_worlds=93, seed=0,
                                                         auto_reset=2))):
        rate, ro, up = train_rate(env)
        print('training, %s (%d agents): %.0f agent-steps/s (rollout %.3f s, update %.3f s per update; mean of '
              'updates 2-4)' % (name, env.N, rate, ro, up), flush=True)
        del env
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
