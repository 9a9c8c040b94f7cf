#!/usr/bin/env python
"""The cost of DESIGN.md §9r's acceleration limits: CUDA-event time of rlca_dynamics_action alone next to
rlca_latency_action (200 launches after a warm-up, replayed from a CUDA graph, best of five replays, and issued eagerly
from Python) at the bench shape (stage 1, 171 worlds x 24 robots) and at 1024 worlds x 16 robots (random K = 16), and
of the evaluation tick (stage2.pth, random K = 16, 1024 worlds) without and with limits drawn in 0.5..2 m/s^2 and
1..4 rad/s^2, alternating, three rounds each.  Prints the card, power limit and max SM clock first.

    python tools/time_dynamics.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200.dynamics import Dynamics, DynamicsParams  # noqa: E402
from rl_collision_avoidance_b200.evaluation import evaluate  # noqa: E402
from rl_collision_avoidance_b200.latency import Latency, LatencyParams  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402
from time_noise import _events  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
RANGED = DynamicsParams(linear=(0.5, 2.0), angular=(1.0, 4.0), seed=1)


def time_kernels(env, launches=200):
    """(dynamics µs, latency action µs) per launch on `env`'s shape, after a tick so the flags are real"""
    dyn = Dynamics(env, RANGED)
    lat = Latency(env, LatencyParams(command_delay=(2, 2), seed=1))
    env.reset_world()
    env.reset_pose()
    stacks = [env.obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, env.beam_mum, device='cuda')]
    cmd = torch.rand(env.N, 2, device='cuda')
    dyn.action(cmd)
    lat.action(cmd)
    env.control_vel(torch.full((env.N, 2), 0.5, device='cuda'), stack_in=stacks[0], stack_out=stacks[1])
    return (_events(lambda: dyn.action(cmd, env.flags), launches),
            _events(lambda: lat.action(cmd, env.flags), launches))


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick without and with limits"""
    env = StageWorld(512, scenario=make_scenario('random', robots_per_world=16), num_worlds=1024, seed=0, auto_reset=0)
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    evaluate(env, pol, 1, 20, check_every=10 ** 9, dynamics=Dynamics(env, RANGED))     # warm-up of every kernel
    out = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            dyn = Dynamics(env, RANGED) if on else None
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            evaluate(env, pol, 1, ticks, check_every=10 ** 9, dynamics=dyn)
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
        d, a = time_kernels(env)
        print('%s: rlca_dynamics_action %.2f us graph-replayed (%.2f us per eager call); rlca_latency_action (delay 2) '
              '%.2f us graph-replayed (%.2f us per eager call)' % (name, d[0], d[1], a[0], a[1]), flush=True)
    off, on = time_ticks()
    print('evaluation tick, random K = 16, 1024 worlds, stage2.pth, ms per tick over 200 ticks, alternating: '
          'without %s | with limits 0.5..2 m/s^2, 1..4 rad/s^2 %s'
          % (' '.join('%.4f' % v for v in off), ' '.join('%.4f' % v for v in on)))


if __name__ == '__main__':
    main()
