#!/usr/bin/env python
"""The cost of DESIGN.md §9u's dynamic-window baseline: CUDA-event time of rlca_dwa_action (200 launches after a
warm-up, replayed from a CUDA graph, best of five replays, and issued eagerly from Python) at the bench shape (stage 1,
171 worlds x 24 robots), at 1024 worlds x 16 robots (random K = 16), on stage 2 (24 worlds x 44 robots) and on the
50-robot circle (24 worlds), each next to the policy's deterministic action (generate_action_no_sampling, stage2.pth,
eager) at the same N; and the evaluation tick (random K = 16, 1024 worlds) driven by DWA and by stage2.pth,
alternating, three rounds each.  Prints the card, power limit and max SM clock first.

    python tools/time_dwa.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from rl_collision_avoidance_b200.dwa import DwaController, DwaParams  # noqa: E402
from rl_collision_avoidance_b200.evaluation import ACTION_BOUND, evaluate  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.model.ppo import generate_action_no_sampling  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402
from time_noise import _events  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def _policy(n):
    pol = CNNPolicy(frames=3, action_space=2, max_batch=n)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    return pol


def _eager(fn, launches):
    for _ in range(20):
        fn()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(launches):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / launches * 1e3


def time_kernels(env, launches=200):
    """(DWA (graph µs, eager µs) with the default grid, DWA with a 5 x 9 grid and window limits, policy eager µs) per
    call after 20 ticks, so the robots are spread and the scans hold returns"""
    env.reset_world()
    env.reset_pose()
    if env.sc.layout is not None:
        env.random_layout()
    stacks = [env.obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, 512, device='cuda')]
    for t in range(20):
        env.control_vel(torch.full((env.N, 2), 0.5, device='cuda'), stack_in=stacks[t & 1],
                        stack_out=stacks[1 - (t & 1)])
    stack = stacks[0]
    dwa = DwaController(env, DwaParams())
    small = DwaController(env, DwaParams(v_samples=5, w_samples=9, accel=2.0, angular_accel=4.0))
    pol = _policy(env.N)
    goal, speed = env.get_local_goal(), env.get_self_speed()
    fallback = None
    dwa(stack, env.gs)
    torch.cuda.synchronize()
    fallback = float(dwa.status().float().mean())
    return (_events(lambda: dwa(stack, env.gs), launches), _events(lambda: small(stack, env.gs), launches),
            _eager(lambda: generate_action_no_sampling(env=env, state_list=(stack, goal, speed), policy=pol,
                                                       action_bound=ACTION_BOUND), launches), fallback)


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick driven by DWA and by stage2.pth"""
    env = StageWorld(512, scenario=make_scenario('random', robots_per_world=16), num_worlds=1024, seed=0, auto_reset=0)
    pol, dwa = _policy(env.N), DwaController(env, DwaParams())
    evaluate(env, pol, 1, 20, check_every=10 ** 9)      # warm-up
    evaluate(env, dwa, 1, 20, check_every=10 ** 9)
    out = {'policy': [], 'dwa': []}
    for _ in range(rounds):
        for name, ctrl in (('policy', pol), ('dwa', dwa)):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            evaluate(env, ctrl, 1, ticks, check_every=10 ** 9)
            t1.record()
            torch.cuda.synchronize()
            out[name].append(t0.elapsed_time(t1) / ticks)
    return out['policy'], out['dwa']


def main():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        q = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), q))
    envs = (('171 x 24 (bench), stage 1', StageWorld(512, scenario='stage1', num_worlds=171, seed=0, auto_reset=1)),
            ('1024 x 16, random layouts', StageWorld(512, scenario=make_scenario('random', robots_per_world=16),
                                                     num_worlds=1024, seed=0, auto_reset=0)),
            ('24 x 44, stage 2', StageWorld(512, scenario='stage2', num_worlds=24, seed=0, auto_reset=2)),
            ('24 x 50, circle', StageWorld(512, scenario='circle', num_worlds=24, seed=0, auto_reset=0)))
    for name, env in envs:
        d, s, p, fb = time_kernels(env)
        print('%s: rlca_dwa_action 11 x 21 %.2f us graph-replayed (%.2f eager); 5 x 9 with limits %.2f us (%.2f '
              'eager); generate_action_no_sampling %.2f us eager; fallback share of the timed call %.4f'
              % (name, d[0], d[1], s[0], s[1], p, fb), flush=True)
    pol, dwa = time_ticks()
    print('evaluation tick, random K = 16, 1024 worlds, ms per tick over 200 ticks, alternating: stage2.pth %s | '
          'DWA %s' % (' '.join('%.4f' % v for v in pol), ' '.join('%.4f' % v for v in dwa)))


if __name__ == '__main__':
    main()
