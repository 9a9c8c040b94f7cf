#!/usr/bin/env python
"""The non-cooperative results of DESIGN.md §9h: evaluate.py with --non-cooperative K for K in {1, 5} on the 50-robot
circle (--episodes 1) and on stage 2 (--episodes 3), 8 worlds, seed 0, for stage2.pth, NH-ORCA+map and ORCA-DD.  Prints
one markdown row per run and role, and the card and power limit they were measured on.

    python tools/noncoop_table.py
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
               ('ORCA-DD', ['--baseline', 'orca'])]


def row(name, scenario, k, role, m):
    f = lambda key: '–' if m[key][0] != m[key][0] else '%.3f ± %.3f' % m[key]
    return '| %s | %s | %d | %s | %d | %.3f | %.3f | %.3f | %d | %s | %s | %s |' % (
        name, scenario, k, role, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
        m['unfinished'], f('extra_time'), f('extra_distance'), f('average_speed'))


def main():
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    print('| controller | scenario | K | role | episodes | success | crash | time-out | unfinished | extra time | '
          'extra distance | average speed |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|')
    for scenario, episodes in (('circle', 1), ('stage2', 3)):
        for name, who in CONTROLLERS:
            for k in (1, 5):
                with contextlib.redirect_stdout(io.StringIO()):
                    out = evaluate.main(['--scenario', scenario, '--num-worlds', '8', '--episodes', str(episodes),
                                         '--seed', '0', '--non-cooperative', str(k)] + who)
                for role in ('cooperative', 'non_cooperative'):
                    print(row(name, scenario, k, role.replace('_', '-'), out['by_role'][role]), flush=True)


if __name__ == '__main__':
    main()
