#!/usr/bin/env python
"""The results of DESIGN.md §9v: evaluate.py --timeouts for stage2.pth, NH-ORCA+map and the dynamic-window baseline on
arenas (64 arenas of 10 m, 4..10 obstacles, arena seed 0, K = 8, one world per arena) and on random layouts (K = 8,
64 worlds), seed 0.  Prints one markdown row per run (time-outs and unfinished episodes split into frozen / stalled /
slow) and the card, power limit and maximum SM clock.  One seed: observations, not effect sizes.

    python tools/arena_table.py
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

CONTROLLERS = [('`stage2.pth`', ['--policy', os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')]),
               ('NH-ORCA+map', ['--baseline', 'nh-orca', '--orca-map']),
               ('DWA', ['--baseline', 'dwa'])]
SCENARIOS = [('arenas, seed 0', ['--scenario', 'arena', '--arena-robots', '8', '--num-worlds', '64']),
             ('arenas, seed 1', ['--scenario', 'arena', '--arena-robots', '8', '--num-worlds', '64',
                                 '--arena-seed', '1']),
             ('random K = 8', ['--scenario', 'random', '--random-robots', '8', '--num-worlds', '64'])]


def row(name, scenario, out):
    m, p = out['metrics'], out['progress']
    f = lambda key: '–' if m[key][0] != m[key][0] else '%.3f ± %.3f' % m[key]
    stuck = lambda g: '%d / %d / %d' % (p[g + '_frozen'], p[g + '_stalled'], p[g + '_slow'])
    return '| %s | %s | %d | %.3f | %.3f | %.3f | %d | %s | %s | %s | %s |' % (
        name, scenario, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'], m['unfinished'],
        stuck('timeout'), stuck('unfinished'), f('extra_time'), f('extra_distance'))


def main():
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info))
    print('| controller | scenario | episodes | success | crash | time-out | unfinished | '
          'time-outs frozen / stalled / slow | unfinished frozen / stalled / slow | extra time | extra distance |')
    print('|---|---|---|---|---|---|---|---|---|---|---|')
    for sname, sargv in SCENARIOS:
        for name, who in CONTROLLERS:
            with contextlib.redirect_stdout(io.StringIO()):
                out = evaluate.main(sargv + who + ['--timeouts', '--seed', '0'])
            print(row(name, sname, out), flush=True)


if __name__ == '__main__':
    main()
