#!/usr/bin/env python
"""The results of DESIGN.md §9w: evaluate.py --timeouts with the global planner on arenas (64 arenas of 10 m, 4..10
obstacles, arena seeds 0 and 1, K = 8, 64 worlds) and on stage 2 (8 worlds, 2 episodes per robot), seed 0:
`stage2.pth` and the dynamic-window baseline each with --geodesic and with --planner, and NH-ORCA+map with --geodesic.
Prints one markdown row per run and the card, power limit and maximum SM clock.  One seed: observations, not effect
sizes.

    python tools/planner_table.py
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

STAGE2 = ['--policy', os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')]
CONTROLLERS = [('`stage2.pth`', STAGE2 + ['--geodesic']), ('`stage2.pth` + planner', STAGE2 + ['--planner']),
               ('DWA', ['--baseline', 'dwa', '--geodesic']), ('DWA + planner', ['--baseline', 'dwa', '--planner']),
               ('NH-ORCA+map', ['--baseline', 'nh-orca', '--orca-map', '--geodesic'])]
SCENARIOS = [('arenas, seed 0', ['--scenario', 'arena', '--arena-robots', '8', '--num-worlds', '64']),
             ('arenas, seed 1', ['--scenario', 'arena', '--arena-robots', '8', '--num-worlds', '64',
                                 '--arena-seed', '1']),
             ('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '2'])]


def row(name, scenario, out):
    m, p, g = out['metrics'], out['progress'], out['geodesic']
    f = lambda v: '–' if v[0] != v[0] else '%.3f ± %.3f' % v
    unf = '%d / %d / %d' % (p['unfinished_frozen'], p['unfinished_stalled'], p['unfinished_slow'])
    pl = out.get('planner')
    shares = '%.3f / %.3f / %.3f' % (pl['goal_visible'], pl['waypoint'], pl['no_plan']) if pl else '–'
    return '| %s | %s | %d | %.3f | %.3f | %.3f | %d (%s) | %s | %s | %s | %d |' % (
        name, scenario, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'], m['unfinished'], unf,
        f(m['extra_distance']), f(g['extra_geodesic_distance']), shares, g['no_path'])


def main():
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info))
    print('| controller | scenario | episodes | success | crash | time-out | unfinished (frozen / stalled / slow) | '
          'extra distance m | extra geodesic distance m | goal visible / waypoint / no plan | no path |')
    print('|---|---|---|---|---|---|---|---|---|---|---|')
    for sname, sargv in SCENARIOS:
        for name, who in CONTROLLERS:
            with contextlib.redirect_stdout(io.StringIO()):
                out = evaluate.main(sargv + who + ['--timeouts', '--seed', '0'])
            print(row(name, sname, out), flush=True)


if __name__ == '__main__':
    main()
