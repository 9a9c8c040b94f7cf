#!/usr/bin/env python
"""The robustness results of DESIGN.md §9s: evaluate.py --safety --timeouts for stage2.pth and stage1_2.pth on stage 2
(8 worlds, 3 episodes per robot) and on random K = 16 (--random-worlds worlds, one episode per robot), seed 0,
localization seed 0, without error, under position errors of 0.1 and 0.3 m alone, heading errors of 0.05 and 0.15 rad
alone (tau 2 s), a 0.1 m position error at tau 0 and inf, speed noise alone (0.05 m/s, 0.1 rad/s), and one combined row
(0.1..0.3 m, 0.05..0.15 rad drawn per robot and episode, tau 2 s, speed noise).  One markdown row per run: success,
crash and time-out rates, extra time (mean +- std over the successful episodes), crashes by cause and the time-outs and
unfinished episodes called frozen / stalled / slow (DESIGN.md §9o).  Prints the card first.

    python tools/localization_table.py [--random-worlds 1024]
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
GRID = [('none', []),
        ('xy 0.1', ['--pose-error', '0.1']), ('xy 0.3', ['--pose-error', '0.3']),
        ('theta 0.05', ['--heading-error', '0.05']), ('theta 0.15', ['--heading-error', '0.15']),
        ('xy 0.1, tau 0', ['--pose-error', '0.1', '--pose-error-time', '0']),
        ('xy 0.1, tau inf', ['--pose-error', '0.1', '--pose-error-time', 'inf']),
        ('speed 0.05, 0.1', ['--speed-error', '0.05,0.1']),
        ('combined', ['--pose-error', '0.1,0.3', '--heading-error', '0.05,0.15', '--speed-error', '0.05,0.1'])]


def _row(who, sname, lname, argv):
    with contextlib.redirect_stdout(io.StringIO()):
        out = evaluate.main(argv)
    m, s, p = out['metrics'], out['safety'], out['progress']
    causes = lambda g: '%d / %d / %d' % (p[g + '_frozen'], p[g + '_stalled'], p[g + '_slow'])
    print('| %s | %s | %s | %d | %.4f | %.4f | %.4f | %.2f +- %.2f | %d / %d | %s | %s |'
          % (who, sname, lname, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
             m['extra_time'][0], m['extra_time'][1], s['crash_static'], s['crash_robot'], causes('timeout'),
             causes('unfinished')), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--random-worlds', type=int, default=1024)
    ap.add_argument('--policies', default='stage2.pth,stage1_2.pth')
    args = ap.parse_args()
    print('card: %s' % torch.cuda.get_device_name(0))
    scen = [('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3']),
            ('random K=16', ['--scenario', 'random', '--random-robots', '16', '--num-worlds', str(args.random_worlds)])]
    print('| policy | scenario | error | episodes | success | crash | time-out | extra time (s) | '
          'crashes static / robot | time-outs frozen / stalled / slow | unfinished frozen / stalled / slow |')
    print('|---|---|---|---|---|---|---|---|---|---|---|')
    for pol in args.policies.split(','):
        for sname, sargs in scen:
            for lname, largs in GRID:
                _row(pol, sname, lname, sargs + ['--policy', os.path.join(CKPT, pol), '--safety', '--timeouts'] + largs)


if __name__ == '__main__':
    main()
