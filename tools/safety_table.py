#!/usr/bin/env python
"""The safety results of DESIGN.md §9m: evaluate.py --safety for the shipped checkpoints, NH-ORCA with the map and
ORCA-DD on stage 2 (8 worlds, 3 episodes), the 50-robot circle (8 worlds, one episode) and random scenarios with K in
{8, 16, 32} robots (default 10 m square, --random-worlds worlds, one episode per robot), seed 0: crashes by cause, minimum
separation and clearance over the successful episodes, near-miss rate.  Then the cost: CUDA-event time of
rlca_safety_track alone (200 launches after a warm-up) at 1024 worlds x 16 robots and 171 worlds x 24 robots, 512
beams, and of the evaluation tick with and without the option, alternating, three rounds each.  Prints the card and
power limit first.

    python tools/safety_table.py [--random-worlds 1024] [--skip-table] [--skip-timing]
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
from rl_collision_avoidance_b200.evaluation import EpisodeTracker, SafetyTracker, evaluate as run_evaluate  # noqa: E402
from rl_collision_avoidance_b200.model.net import CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
CONTROLLERS = [('`%s`' % f, ['--policy', os.path.join(CKPT, f)]) for f in ('stage2.pth', 'stage1_2.pth', 'stage1_1.pth')] + \
              [('NH-ORCA+map', ['--baseline', 'nh-orca', '--orca-map']), ('ORCA-DD', ['--baseline', 'orca'])]


def runs(random_worlds):
    return [('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3']),
            ('circle', ['--scenario', 'circle', '--num-worlds', '8', '--episodes', '1'])] + \
           [('random K = %d' % K, ['--scenario', 'random', '--random-robots', str(K), '--num-worlds', str(random_worlds)])
            for K in (8, 16, 32)]


def row(name, scenario, out):
    m, s = out['metrics'], out['safety']
    f = lambda v: '–' if v[0] != v[0] else '%.3f ± %.3f' % v
    near = '–' if s['near_miss_rate'] != s['near_miss_rate'] else '%.3f' % s['near_miss_rate']
    return '| %s | %s | %d | %d | %.3f | %.3f | %d | %d | %d | %s | %s | %s | %.3f |' % (
        name, scenario, out['partials'].shape[0], m['episodes'], m['success_rate'], m['crash_rate'], s['crash_static'],
        s['crash_robot'], s['crash_both_in_range'], f(s['min_separation_reached']), f(s['min_clearance_reached']),
        near, s['min_separation'])


def table(random_worlds):
    print('| controller | scenario | worlds | episodes | success | crash | static | robot | both in range | '
          'min separation, m | min clearance, m | near-miss rate | least separation, m |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|---|')
    for scenario, run in runs(random_worlds):
        for name, who in CONTROLLERS:
            with contextlib.redirect_stdout(io.StringIO()):
                out = evaluate.main(run + ['--seed', '0', '--safety'] + who)
            print(row(name, scenario, out), flush=True)
            del out
            torch.cuda.empty_cache()


def time_track(sc, worlds, auto_reset, launches=200):
    """Milliseconds per rlca_safety_track launch on the state 20 random-action ticks leave."""
    env = StageWorld(512, scenario=sc, num_worlds=worlds, seed=0, auto_reset=auto_reset)
    env.reset_pose()
    if sc.layout is not None:
        env.random_layout()
    tr = EpisodeTracker(env, 1)
    st = SafetyTracker(env, tr, 0.1)
    rng = np.random.default_rng(0)
    for _ in range(20):
        act = np.stack([rng.uniform(0, 1, env.N), rng.uniform(-1, 1, env.N)], 1).astype(np.float32)
        env.control_vel(torch.from_numpy(act).cuda())
        st.track()
        tr.track()
    tr.reset()                                                     # every robot tracked again: all pairs are computed
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(20):
        st.track()
    t0.record()
    for _ in range(launches):
        st.track()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / launches


def time_ticks(ticks=200, rounds=3):
    """Milliseconds per evaluation tick (stage2.pth, random K = 16, 1024 worlds) without and with the option."""
    sc = make_scenario('random', robots_per_world=16)
    env = StageWorld(512, scenario=sc, num_worlds=1024, seed=0, auto_reset=0)
    pol = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
    pol.load_state_dict(torch.load(os.path.join(CKPT, 'stage2.pth'), map_location='cuda'))
    run_evaluate(env, pol, 1, 20, check_every=10 ** 9, safety=0.1)            # warm-up of every kernel involved
    out = {None: [], 0.1: []}
    for _ in range(rounds):
        for safety in (None, 0.1):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            run_evaluate(env, pol, 1, ticks, check_every=10 ** 9, safety=safety)
            t1.record()
            torch.cuda.synchronize()
            out[safety].append(t0.elapsed_time(t1) / ticks)
    return out[None], out[0.1]


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
        b = time_track(make_scenario('stage1'), 171, 1)
        print('rlca_safety_track alone: %.4f ms at 1024 worlds x 16 robots x 512 beams, %.4f ms at 171 x 24 x 512' % (a, b))
        off, on = time_ticks()
        print('evaluation tick, random K = 16, 1024 worlds, stage2.pth, ms per tick over 200 ticks, alternating: '
              'without %s | with --safety %s' % (' '.join('%.4f' % v for v in off), ' '.join('%.4f' % v for v in on)))
    if not args.skip_table:
        table(args.random_worlds)


if __name__ == '__main__':
    main()
