#!/usr/bin/env python
"""The cost of DESIGN.md §9t's crowd: CUDA-event time of rlca_crowd_action (200 launches after a warm-up, replayed from
a CUDA graph, best of five replays, and issued eagerly from Python) next to rlca_noncoop_action at the bench shape
(stage 1, 171 worlds x 24 robots), at 1024 worlds x 16 robots (random K = 16) and on stage 2 (24 worlds x 44 robots),
map-blind and with the scenario's own map, for 1 and 5 crowd agents per world; and the evaluation tick (stage2.pth,
random K = 16, 1024 worlds) without a crowd and with 5 crowd agents per world on the map, alternating, three rounds
each.  Prints the card, power limit and max SM clock first.

    python tools/time_crowd.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from rl_collision_avoidance_b200.crowd import Crowd  # noqa: E402
from rl_collision_avoidance_b200.evaluation import evaluate, non_cooperative_mask  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.orca import NonCooperative, ObstacleSet  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402
from time_noise import _events  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')


def time_kernels(env, k, launches=200):
    """(crowd map-blind, crowd with the map, non-cooperative), each (graph µs, eager µs) per launch, for k masked
    agents per world, after 20 ticks so the agents are spread"""
    env.reset_world()
    env.reset_pose()
    if env.sc.layout is not None:
        env.random_layout()
    for _ in range(20):
        env.control_vel(torch.full((env.N, 2), 0.5, device='cuda'))
    mask = non_cooperative_mask(env.cfg.robots_per_world, env.num_worlds, k)
    obs = ObstacleSet(env.cfg, env.sc.map.cells, 1.0)
    blind, mapped, nc = Crowd(env, mask), Crowd(env, mask, obstacles=obs), NonCooperative(env, mask)
    act = torch.rand(env.N, 2, device='cuda')
    return (_events(lambda: blind.apply(act), launches), _events(lambda: mapped.apply(act), launches),
            _events(lambda: nc.apply(act), launches))


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick without and with 5 crowd agents per world on the map"""
    env = StageWorld(512, scenario=make_scenario('random', robots_per_world=16), num_worlds=1024, seed=0, auto_reset=0)
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    crowd = Crowd(env, non_cooperative_mask(16, 1024, 5), obstacles=True)
    evaluate(env, pol, 1, 20, check_every=10 ** 9, crowd=crowd)     # warm-up
    out = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            evaluate(env, pol, 1, ticks, check_every=10 ** 9, crowd=crowd if on else None)
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
    envs = (('171 x 24 (bench), stage 1', StageWorld(512, scenario='stage1', num_worlds=171, seed=0, auto_reset=1)),
            ('1024 x 16, random layouts', StageWorld(512, scenario=make_scenario('random', robots_per_world=16),
                                                     num_worlds=1024, seed=0, auto_reset=0)),
            ('24 x 44, stage 2', StageWorld(512, scenario='stage2', num_worlds=24, seed=0, auto_reset=2)))
    for name, env in envs:
        for k in (1, 5):
            b, m, n = time_kernels(env, k)
            print('%s, %d crowd agents per world: rlca_crowd_action map-blind %.2f us graph-replayed (%.2f eager), '
                  'with the map %.2f us (%.2f eager); rlca_noncoop_action %.2f us (%.2f eager)'
                  % (name, k, b[0], b[1], m[0], m[1], n[0], n[1]), flush=True)
    off, on = time_ticks()
    print('evaluation tick, random K = 16, 1024 worlds, stage2.pth, ms per tick over 200 ticks, alternating: '
          'without %s | with 5 crowd agents per world on the map %s'
          % (' '.join('%.4f' % v for v in off), ' '.join('%.4f' % v for v in on)))


if __name__ == '__main__':
    main()
