#!/usr/bin/env python
"""The robustness results of DESIGN.md §9r: evaluate.py --safety for stage2.pth and stage1_2.pth on stage 2 (8 worlds,
3 episodes per robot) and on random K = 16 (--random-worlds worlds, one episode per robot), seed 0, dynamics seed 0,
without limits, under linear limits of 2, 1 and 0.5 m/s^2 alone, angular limits of 4 and 2 rad/s^2 alone, both (1, 2)
and both drawn per robot and episode (0.5..2, 1..4); and NH-ORCA with the map on stage 2 without limits and at (1, 2).
One markdown row per run: success, crash and time-out rates, extra time (mean +- std over the successful episodes) and
crashes by cause.  Prints the card first.

    python tools/dynamics_table.py [--random-worlds 1024]
"""
import argparse
import contextlib
import io
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import evaluate  # noqa: E402

CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')
BOTH = ('both 1, 2', ['--accel-limit', '1', '--angular-accel-limit', '2'])
GRID = [('none', [])] + [('linear %g' % a, ['--accel-limit', str(a)]) for a in (2, 1, 0.5)] + \
    [('angular %g' % b, ['--angular-accel-limit', str(b)]) for b in (4, 2)] + \
    [BOTH, ('ranged 0.5..2, 1..4', ['--accel-limit', '0.5,2', '--angular-accel-limit', '1,4'])]


def _row(who, sname, lname, argv):
    with contextlib.redirect_stdout(io.StringIO()):
        out = evaluate.main(argv)
    m, s = out['metrics'], out['safety']
    print('| %s | %s | %s | %d | %.4f | %.4f | %.4f | %.2f +- %.2f | %d / %d |'
          % (who, sname, lname, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
             m['extra_time'][0], m['extra_time'][1], s['crash_static'], s['crash_robot']), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--random-worlds', type=int, default=1024)
    ap.add_argument('--policies', default='stage2.pth,stage1_2.pth')
    args = ap.parse_args()
    print('card: %s' % torch.cuda.get_device_name(0))
    stage2 = ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3']
    scen = [('stage 2', stage2),
            ('random K=16', ['--scenario', 'random', '--random-robots', '16', '--num-worlds', str(args.random_worlds)])]
    print('| controller | scenario | limits (m/s^2, rad/s^2) | episodes | success | crash | time-out | '
          'extra time (s) | crashes static / robot |')
    print('|---|---|---|---|---|---|---|---|---|')
    for pol in args.policies.split(','):
        for sname, sargs in scen:
            for lname, largs in GRID:
                _row(pol, sname, lname, sargs + ['--policy', os.path.join(CKPT, pol), '--safety'] + largs)
    for lname, largs in (GRID[0], BOTH):
        _row('NH-ORCA + map', 'stage 2', lname, stage2 + ['--baseline', 'nh-orca', '--orca-map', '--safety'] + largs)


if __name__ == '__main__':
    main()
