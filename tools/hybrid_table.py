#!/usr/bin/env python
"""The hybrid-controller results of DESIGN.md §9j: evaluate.py for stage2.pth alone, with the hybrid at its defaults,
with the driver only (RL+driver: r_risk = 0) and with the speed cap only (RL+safe: r_safe = range_max), on random
scenarios with K in {8, 16, 32} robots (default 10 m square, 1024 worlds, one episode per robot), on the 50-robot
circle (8 worlds, one episode) and on stage 2 (8 worlds, 3 episodes), seed 0.  Prints the card and power limit, then
one markdown row per run with the share of counted robot-ticks in each mode.

    python tools/hybrid_table.py
"""
import contextlib
import io
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import evaluate  # noqa: E402
from rl_collision_avoidance_b200.scenarios import COMMON  # noqa: E402

POLICY = ['--policy', os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')]
CONTROLLERS = [('`stage2.pth`', POLICY),
               ('hybrid', POLICY + ['--hybrid']),
               ('RL+driver', POLICY + ['--hybrid', '--hybrid-r-risk', '0']),
               ('RL+safe', POLICY + ['--hybrid', '--hybrid-r-safe', repr(COMMON['range_max'])])]
RUNS = [('random K = %d' % K, ['--scenario', 'random', '--random-robots', str(K), '--num-worlds', '1024'])
        for K in (8, 16, 32)] + \
       [('circle', ['--scenario', 'circle', '--num-worlds', '8', '--episodes', '1']),
        ('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3'])]


def row(name, scenario, out):
    m = out['metrics']
    f = lambda key: '–' if m[key][0] != m[key][0] else '%.3f ± %.3f' % m[key]
    s = out.get('modes')
    shares = ' | '.join('%.3f' % s[k] for k in ('policy', 'driver', 'safe')) if s else '– | – | –'
    return '| %s | %s | %d | %d | %d | %.3f | %.3f | %.3f | %d | %s | %s | %s | %s |' % (
        name, scenario, out['partials'].shape[0], out['ticks'], m['episodes'], m['success_rate'], m['crash_rate'],
        m['timeout_rate'], m['unfinished'], f('extra_time'), f('extra_distance'), f('average_speed'), shares)


def main():
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    print('| controller | scenario | worlds | ticks | episodes | success | crash | time-out | unfinished | extra time | '
          'extra distance | average speed | policy | driver | safe |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|')
    for scenario, run in RUNS:
        for name, who in CONTROLLERS:
            with contextlib.redirect_stdout(io.StringIO()):
                out = evaluate.main(run + ['--seed', '0'] + who)
            print(row(name, scenario, out), flush=True)
            del out
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
