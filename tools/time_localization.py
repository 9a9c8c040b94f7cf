#!/usr/bin/env python
"""The cost of DESIGN.md §9s's localization error: CUDA-event time of rlca_localization_observe alone next to
rlca_dynamics_action (200 launches after a warm-up, replayed from a CUDA graph, best of five replays, and issued eagerly
from Python) at the bench shape (stage 1, 171 worlds x 24 robots) and at 1024 worlds x 16 robots (random K = 16), and
of the evaluation tick (stage2.pth, random K = 16, 1024 worlds) without and with pose, heading and speed error,
alternating, three rounds each.  Prints the card, power limit and max SM clock first.

    python tools/time_localization.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200.dynamics import Dynamics, DynamicsParams  # noqa: E402
from rl_collision_avoidance_b200.evaluation import evaluate  # noqa: E402
from rl_collision_avoidance_b200.localization import Localization, LocalizationParams  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402
from time_noise import _events  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
RANGED = LocalizationParams(pose_sigma=(0.1, 0.3), heading_sigma=(0.05, 0.15), correlation_time=2.0,
                            speed_sigma=(0.05, 0.1), seed=1)


def time_kernels(env, launches=200):
    """(localization µs, dynamics µs) per launch on `env`'s shape, after a tick so the flags are real"""
    loc = Localization(env, RANGED)
    dyn = Dynamics(env, DynamicsParams(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=1))
    env.reset_world()
    env.reset_pose()
    stacks = [env.obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, env.beam_mum, device='cuda')]
    cmd = torch.rand(env.N, 2, device='cuda')
    loc.observe()
    dyn.action(cmd)
    env.control_vel(torch.full((env.N, 2), 0.5, device='cuda'), stack_in=stacks[0], stack_out=stacks[1])
    return (_events(lambda: loc.observe(env.flags), launches),
            _events(lambda: dyn.action(cmd, env.flags), launches))


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick without and with localization error"""
    env = StageWorld(512, scenario=make_scenario('random', robots_per_world=16), num_worlds=1024, seed=0, auto_reset=0)
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    evaluate(env, pol, 1, 20, check_every=10 ** 9, localization=Localization(env, RANGED))     # warm-up
    out = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            loc = Localization(env, RANGED) if on else None
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            evaluate(env, pol, 1, ticks, check_every=10 ** 9, localization=loc)
            t1.record()
            torch.cuda.synchronize()
            out[on].append(t0.elapsed_time(t1) / ticks)
    return out[False], out[True]


def main():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        q = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), q))
    bench = StageWorld(512, scenario='stage1', num_worlds=171, seed=0, auto_reset=1)
    big = StageWorld(512, scenario=make_scenario('random', robots_per_world=16), num_worlds=1024, seed=0, auto_reset=0)
    for name, env in (('171 x 24 (bench)', bench), ('1024 x 16', big)):
        o, d = time_kernels(env)
        print('%s: rlca_localization_observe %.2f us graph-replayed (%.2f us per eager call); rlca_dynamics_action '
              '%.2f us graph-replayed (%.2f us per eager call)' % (name, o[0], o[1], d[0], d[1]), flush=True)
    off, on = time_ticks()
    print('evaluation tick, random K = 16, 1024 worlds, stage2.pth, ms per tick over 200 ticks, alternating: '
          'without %s | with pose 0.1..0.3 m, heading 0.05..0.15 rad, tau 2 s, speed 0.05, 0.1 %s'
          % (' '.join('%.4f' % v for v in off), ' '.join('%.4f' % v for v in on)))


if __name__ == '__main__':
    main()
