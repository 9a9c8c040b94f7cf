#!/usr/bin/env python
"""The robustness results of DESIGN.md §9q: evaluate.py --safety for stage1_2.pth and stage2.pth on stage 2 (8 worlds,
3 episodes per robot) and on random K = 16 (--random-worlds worlds, one episode per robot), seed 0, latency seed 0,
over scan delays of 1, 2 and 4 ticks, command delays of 1, 2 and 4 ticks, both at 2, and both drawn in 0..4 per robot
and episode (one tick is 0.1 s).  One markdown row per run: success, crash and time-out rates, extra time (mean +- std
over the successful episodes) and crashes by cause.  Prints the card first.

    python tools/latency_table.py [--random-worlds 1024]
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
GRID = [('none', [])] + [('scan %d' % d, ['--scan-delay', str(d)]) for d in (1, 2, 4)] + \
    [('command %d' % d, ['--command-delay', str(d)]) for d in (1, 2, 4)] + \
    [('both 2', ['--scan-delay', '2', '--command-delay', '2']),
     ('both 0..4', ['--scan-delay', '0,4', '--command-delay', '0,4'])]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--random-worlds', type=int, default=1024)
    ap.add_argument('--policies', default='stage2.pth,stage1_2.pth')
    args = ap.parse_args()
    print('card: %s' % torch.cuda.get_device_name(0))
    scen = [('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3']),
            ('random K=16', ['--scenario', 'random', '--random-robots', '16', '--num-worlds', str(args.random_worlds)])]
    print('| policy | scenario | latency (ticks) | episodes | success | crash | time-out | extra time (s) | '
          'crashes static / robot |')
    print('|---|---|---|---|---|---|---|---|---|')
    for pol in args.policies.split(','):
        for sname, sargs in scen:
            for lname, largs in GRID:
                argv = sargs + ['--policy', os.path.join(CKPT, pol), '--safety'] + largs
                with contextlib.redirect_stdout(io.StringIO()):
                    out = evaluate.main(argv)
                m, s = out['metrics'], out['safety']
                print('| %s | %s | %s | %d | %.4f | %.4f | %.4f | %.2f +- %.2f | %d / %d |'
                      % (pol, sname, lname, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
                         m['extra_time'][0], m['extra_time'][1], s['crash_static'], s['crash_robot']), flush=True)


if __name__ == '__main__':
    main()
