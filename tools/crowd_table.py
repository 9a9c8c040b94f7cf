#!/usr/bin/env python
"""The crowd results of DESIGN.md §9t: evaluate.py with K in {1, 5} masked agents per world on stage 2 (8 worlds,
--episodes 3), the 50-robot circle (8 worlds) and random layouts (K = 16 robots, 64 worlds), seed 0, for stage2.pth and
NH-ORCA+map, the masked agents being a crowd that sees the robots, a crowd that ignores them (both with --crowd-map)
or §9h's straight drivers.  Prints one markdown row per run and role, and the card and power limit.

With --checkpoints NAME=PATH,... the policies given instead, on stage 2 and on random layouts, without masked agents
and with 4 crowd agents per world (the fine-tune comparison of §9t).

    python tools/crowd_table.py
    python tools/crowd_table.py --checkpoints ft=policy/stage2_100.pth
"""
import argparse
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
               ('NH-ORCA+map', ['--baseline', 'nh-orca', '--orca-map'])]
SCENARIOS = [('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3']),
             ('circle', ['--scenario', 'circle', '--num-worlds', '8']),
             ('random K = 16', ['--scenario', 'random', '--random-robots', '16', '--num-worlds', '64'])]
KINDS = [('crowd', ['--crowd-map'], 'crowd'),
         ('crowd ignoring robots', ['--crowd-map', '--crowd-ignores-robots'], 'crowd'),
         ('straight (§9h)', [], 'non_cooperative')]


def row(name, scenario, kind, k, role, m):
    f = lambda key: '–' if m[key][0] != m[key][0] else '%.3f ± %.3f' % m[key]
    return '| %s | %s | %s | %s | %s | %d | %.3f | %.3f | %.3f | %d | %s |' % (
        name, scenario, kind, k, role, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
        m['unfinished'], f('extra_time'))


def run(argv):
    with contextlib.redirect_stdout(io.StringIO()):
        return evaluate.main(argv + ['--seed', '0'])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--checkpoints', default=None, metavar='NAME=PATH,...')
    args = ap.parse_args()
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    print('| controller | scenario | masked | K | role | episodes | success | crash | time-out | unfinished | '
          'extra time |')
    print('|---|---|---|---|---|---|---|---|---|---|---|')
    if args.checkpoints:
        for item in args.checkpoints.split(','):
            name, path = item.split('=')
            for sname, sargv in SCENARIOS[0:3:2]:
                out = run(sargv + ['--policy', path])
                print(row(name, sname, 'none', '–', 'all', out['metrics']), flush=True)
                out = run(sargv + ['--policy', path, '--crowd', '4', '--crowd-map'])
                for role in ('cooperative', 'crowd'):
                    print(row(name, sname, 'crowd', 4, role, out['by_role'][role]), flush=True)
        return
    for sname, sargv in SCENARIOS:
        for name, who in CONTROLLERS:
            for kind, extra, role_key in KINDS:
                for k in (1, 5):
                    flag = '--crowd' if role_key == 'crowd' else '--non-cooperative'
                    out = run(sargv + who + [flag, str(k)] + extra)
                    for role in ('cooperative', role_key):
                        print(row(name, sname, kind, k, role.replace('_', '-'), out['by_role'][role]), flush=True)


if __name__ == '__main__':
    main()
