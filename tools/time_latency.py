#!/usr/bin/env python
"""The cost of DESIGN.md §9q's latency: CUDA-event time of rlca_latency_scan and rlca_latency_action alone (200
launches after a warm-up, replayed from a CUDA graph, best of five replays, and issued eagerly from Python) at the bench
shape (stage 1, 171 worlds x 24 robots x 512 beams) and at 1024 worlds x 16 robots (random K = 16), with both delays 2
and 8, and of the evaluation tick (stage2.pth, random K = 16, 1024 worlds) without and with scan and command delays of
(0, 4) ticks, alternating, three rounds each.  The scan kernel's floor is the data sheet's 3.35 TB/s over the four
frame-sized transfers a row that does not start an episode makes (newest read, ring slot written, ring slot read,
newest written); it is a bound, not a measurement.  Prints the card, power limit and max SM clock first.

    python tools/time_latency.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200.evaluation import evaluate  # noqa: E402
from rl_collision_avoidance_b200.latency import Latency, LatencyParams  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402
from time_noise import _events  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
HBM_BYTES_PER_S = 3.35e12                # H100 SXM data sheet
RANGED = LatencyParams(scan_delay=(0, 4), command_delay=(0, 4), seed=1)


def time_kernels(env, delay, launches=200):
    """(scan µs, action µs) of one launch each on `env`'s shape, with both delays `delay`, after a tick so the flags
    are real"""
    lat = Latency(env, LatencyParams(scan_delay=(delay, delay), command_delay=(delay, delay), seed=1))
    env.reset_world()
    env.reset_pose()
    stacks = [env.obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, env.beam_mum, device='cuda')]
    lat.scan(stacks[0])
    cmd = torch.rand(env.N, 2, device='cuda')
    lat.action(cmd)
    env.control_vel(torch.full((env.N, 2), 0.5, device='cuda'), stack_in=stacks[0], stack_out=stacks[1])
    return (_events(lambda: lat.scan(stacks[1], env.flags), launches),
            _events(lambda: lat.action(cmd, env.flags), launches))


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick without and with latency"""
    env = StageWorld(512, scenario=make_scenario('random', robots_per_world=16), num_worlds=1024, seed=0, auto_reset=0)
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    evaluate(env, pol, 1, 20, check_every=10 ** 9, latency=Latency(env, RANGED))     # warm-up of every kernel involved
    out = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            lat = Latency(env, RANGED) if on else None
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            evaluate(env, pol, 1, ticks, check_every=10 ** 9, latency=lat)
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
        frame = env.N * 512 * 4
        floor_us = 4 * frame / HBM_BYTES_PER_S * 1e6
        for delay in (2, 8):
            s, a = time_kernels(env, delay)
            print('%s, delays %d: rlca_latency_scan %.2f us graph-replayed (%.2f us per eager call), %.1f MB moved, '
                  'data-sheet floor %.2f us, %.0f %% of it achieved; rlca_latency_action %.2f us graph-replayed '
                  '(%.2f us per eager call)'
                  % (name, delay, s[0], s[1], 4 * frame / 1e6, floor_us, 100 * floor_us / s[0], a[0], a[1]), flush=True)
    off, on = time_ticks()
    print('evaluation tick, random K = 16, 1024 worlds, stage2.pth, ms per tick over 200 ticks, alternating: '
          'without %s | with scan and command delay 0..4 %s'
          % (' '.join('%.4f' % v for v in off), ' '.join('%.4f' % v for v in on)))


if __name__ == '__main__':
    main()
