#!/usr/bin/env python
"""The robustness results of DESIGN.md §9p: evaluate.py --safety for stage1_2.pth and stage2.pth on stage 2 (8 worlds,
3 episodes per robot) and on random K = 16 (--random-worlds worlds, one episode per robot), seed 0, noise seed 0, over
a small grid swept one kind at a time (the others at 0): range noise sigma_r in {0, 0.05, 0.1, 0.2} m, beam dropout
p in {0.1, 0.3}, actuation noise sigma_v = sigma_w in {0.1, 0.2}.  One markdown row per run: success, crash and
time-out rates, extra time (mean +- std over the successful episodes) and crashes by cause.  Prints the card first.

    python tools/noise_table.py [--random-worlds 1024]
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
GRID = [('none', [])] + [('sigma_r %g' % s, ['--scan-noise', str(s)]) for s in (0.05, 0.1, 0.2)] + \
    [('p %g' % p, ['--beam-dropout', str(p)]) for p in (0.1, 0.3)] + \
    [('sigma_v,w %g' % s, ['--action-noise', str(s)]) for s in (0.1, 0.2)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--random-worlds', type=int, default=1024)
    args = ap.parse_args()
    print('card: %s' % torch.cuda.get_device_name(0))
    scen = [('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3']),
            ('random K=16', ['--scenario', 'random', '--random-robots', '16', '--num-worlds', str(args.random_worlds)])]
    print('| policy | scenario | noise | episodes | success | crash | time-out | extra time (s) | crashes static / robot |')
    print('|---|---|---|---|---|---|---|---|---|')
    for pol in ('stage1_2.pth', 'stage2.pth'):
        for sname, sargs in scen:
            for nname, nargs in GRID:
                argv = sargs + ['--policy', os.path.join(CKPT, pol), '--safety'] + nargs
                with contextlib.redirect_stdout(io.StringIO()):
                    out = evaluate.main(argv)
                m, s = out['metrics'], out['safety']
                print('| %s | %s | %s | %d | %.4f | %.4f | %.4f | %.2f +- %.2f | %d / %d |'
                      % (pol, sname, nname, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
                         m['extra_time'][0], m['extra_time'][1], s['crash_static'], s['crash_robot']), flush=True)


if __name__ == '__main__':
    main()
