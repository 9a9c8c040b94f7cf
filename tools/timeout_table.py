#!/usr/bin/env python
"""The progress results of DESIGN.md §9o: evaluate.py --timeouts for the shipped checkpoints on stage 1, stage 2 and
the 50-robot circle (the §9c commands: 8 worlds, 3 episodes on the stages and one on the circle), stage2.pth on random
scenarios with K in {16, 32} robots (default 10 m square, --random-worlds worlds, one episode per robot), and
NH-ORCA with the map and ORCA-DD on stage 2 and the circle, seed 0: why the time-outs and the unfinished episodes
failed (frozen / stalled / slow, and with a robot near), how close to the goal they came, the share of still ticks.
Then the cost: CUDA-event time of rlca_progress_track alone (200 launches after a warm-up) at 1024 worlds x 16 robots,
and of the evaluation tick with and without the option, alternating, three rounds each.  Prints the card and power
limit first.

    python tools/timeout_table.py [--random-worlds 1024] [--skip-table] [--skip-timing]
"""
import argparse
import contextlib
import io
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import evaluate  # noqa: E402
from rl_collision_avoidance_b200.evaluation import EpisodeTracker, ProgressTracker, evaluate as run_evaluate  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
STAGE = {'stage 1': ['--scenario', 'stage1', '--num-worlds', '8', '--episodes', '3'],
         'stage 2': ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3'],
         'circle': ['--scenario', 'circle', '--num-worlds', '8', '--episodes', '1']}
BASELINES = [('NH-ORCA+map', ['--baseline', 'nh-orca', '--orca-map']), ('ORCA-DD', ['--baseline', 'orca'])]


def runs(random_worlds):
    out = []
    for f in ('stage1_1.pth', 'stage1_2.pth', 'stage2.pth'):
        for scenario, run in STAGE.items():
            out.append(('`%s`' % f, scenario, run + ['--policy', os.path.join(CKPT, f)]))
    for K in (16, 32):
        out.append(('`stage2.pth`', 'random K = %d' % K, ['--scenario', 'random', '--random-robots', str(K),
                                                          '--num-worlds', str(random_worlds), '--policy',
                                                          os.path.join(CKPT, 'stage2.pth')]))
    for name, who in BASELINES:
        for scenario in ('stage 2', 'circle'):
            out.append((name, scenario, STAGE[scenario] + who))
    return out


def row(name, scenario, out):
    m, p = out['metrics'], out['progress']
    f = lambda v: '–' if v[0] != v[0] else '%.2f ± %.2f' % v
    share = lambda v: '–' if v != v else '%.2f' % v
    group = lambda g, n: '%d | %s | %s | %s | %s | %s' % (
        n, share(p[g + '_frozen_share']), share(p[g + '_stalled_share']), share(p[g + '_slow_share']),
        share(p[g + '_robot_near_share']), f(p[g + '_closest']))
    return '| %s | %s | %d | %.3f | %s | %s | %s |' % (
        name, scenario, m['episodes'], m['timeout_rate'], group('timeout', p['timeouts']),
        group('unfinished', p['unfinished']), share(p['still_share']))


def table(random_worlds):
    print('| controller | scenario | episodes | time-out rate | time-outs | frozen | stalled | slow | robot near | '
          'closest, m | unfinished | frozen | stalled | slow | robot near | closest, m | still share |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|')
    for name, scenario, run in runs(random_worlds):
        with contextlib.redirect_stdout(io.StringIO()):
            out = evaluate.main(run + ['--seed', '0', '--timeouts'])
        print(row(name, scenario, out), flush=True)
        del out
        torch.cuda.empty_cache()


def time_track(sc, worlds, auto_reset, launches=200):
    """Milliseconds per rlca_progress_track launch on the state 20 random-action ticks leave."""
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=0, auto_reset=auto_reset)
    env.reset_pose()
    if sc.layout is not None:
        env.random_layout()
    tr = EpisodeTracker(env, 1)
    pt = ProgressTracker(env, tr)
    rng = np.random.default_rng(0)
    for _ in range(20):
        act = np.stack([rng.uniform(0, 1, env.N), rng.uniform(-1, 1, env.N)], 1).astype(np.float32)
        env.control_vel(torch.from_numpy(act).cuda())
        pt.track()
        tr.track()
    tr.reset()                                                     # every robot tracked again
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(20):
        pt.track()
    t0.record()
    for _ in range(launches):
        pt.track()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / launches


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick (stage2.pth, random K = 16, 1024 worlds) without and with the option."""
    sc = make_scenario('random', robots_per_world=16)
    env = StageWorld(512, scenario=sc, num_worlds=1024, seed=0, auto_reset=0)
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    run_evaluate(env, pol, 1, 20, check_every=10 ** 9, progress={})          # warm-up of every kernel involved
    out = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            run_evaluate(env, pol, 1, ticks, check_every=10 ** 9, progress={} if on else None)
            t1.record()
            torch.cuda.synchronize()
            out[on].append(t0.elapsed_time(t1) / ticks)
    return out[False], out[True]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--random-worlds', type=int, default=1024)
    ap.add_argument('--skip-table', action='store_true')
    ap.add_argument('--skip-timing', action='store_true')
    args = ap.parse_args()
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    if not args.skip_timing:
        a = time_track(make_scenario('random', robots_per_world=16), 1024, 0)
        print('rlca_progress_track alone: %.4f ms at 1024 worlds x 16 robots' % a)
        off, on = time_ticks()
        print('evaluation tick, random K = 16, 1024 worlds, stage2.pth, ms per tick over 200 ticks, alternating: '
              'without %s | with --timeouts %s' % (' '.join('%.4f' % v for v in off), ' '.join('%.4f' % v for v in on)))
    if not args.skip_table:
        table(args.random_worlds)


if __name__ == '__main__':
    main()
