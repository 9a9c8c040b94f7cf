#!/usr/bin/env python
"""The cost of DESIGN.md §9p's noise: CUDA-event time of rlca_noise_scan and rlca_noise_action alone (200 launches after
a warm-up, replayed from a CUDA graph and issued eagerly from Python) at the bench shape (stage 1, 171 worlds x 24
robots x 512 beams) and at 1024 worlds x 16 robots (random K = 16), and of the evaluation tick (stage2.pth, random K = 16, 1024 worlds) without and with every kind of noise on,
alternating, three rounds each.  Prints the card and power limit first.

    python tools/time_noise.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200.evaluation import evaluate  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.noise import Noise, NoiseParams  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
ALL = NoiseParams(range_sigma=0.1, dropout=0.1, v_gain_sigma=0.1, w_gain_sigma=0.1, seed=1)


def _events(fn, launches):
    """(µs per launch replayed from a CUDA graph of `launches` calls: the kernel alone, best of five replays;
    µs per call issued from Python: what an eager loop pays)"""
    for _ in range(20):
        fn()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(launches):
        fn()
    t1.record()
    torch.cuda.synchronize()
    eager = t0.elapsed_time(t1) / launches * 1e3
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            fn()
    g.replay()
    best = float('inf')
    for _ in range(5):
        t0.record()
        g.replay()
        t1.record()
        torch.cuda.synchronize()
        best = min(best, t0.elapsed_time(t1) / launches * 1e3)
    return best, eager


def time_kernels(env, launches=200):
    """(scan µs, action µs) of one launch each on `env`'s shape, after a tick so the flags are real"""
    noise = Noise(env, ALL)
    env.reset_world()
    env.reset_pose()
    stacks = [env.obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(env.N, 3, env.beam_mum, device='cuda')]
    env.control_vel(torch.full((env.N, 2), 0.5, device='cuda'), stack_in=stacks[0], stack_out=stacks[1])
    cmd = torch.rand(env.N, 2, device='cuda')
    return (_events(lambda: noise.scan(stacks[1], env.flags), launches),
            _events(lambda: noise.action(cmd), launches))


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick without and with noise"""
    env = StageWorld(512, scenario=make_scenario('random', robots_per_world=16), num_worlds=1024, seed=0, auto_reset=0)
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    evaluate(env, pol, 1, 20, check_every=10 ** 9, noise=Noise(env, ALL))          # warm-up of every kernel involved
    out = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            noise = Noise(env, ALL) if on else None
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            evaluate(env, pol, 1, ticks, check_every=10 ** 9, noise=noise)
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
        s, a = time_kernels(env)
        mb = env.N * 512 * 4 / 1e6
        print('%s: rlca_noise_scan %.2f us graph-replayed, %.2f us per eager call (newest frame %.1f MB read + '
              'written; fresh rows write 2x more); rlca_noise_action %.2f us graph-replayed, %.2f us per eager call'
              % (name, s[0], s[1], mb, a[0], a[1]))
    off, on = time_ticks()
    print('evaluation tick, random K = 16, 1024 worlds, stage2.pth, ms per tick over 200 ticks, alternating: '
          'without %s | with all noise %s' % (' '.join('%.4f' % v for v in off), ' '.join('%.4f' % v for v in on)))


if __name__ == '__main__':
    main()
