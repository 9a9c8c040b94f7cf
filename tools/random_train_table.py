#!/usr/bin/env python
"""The fine-tune table of DESIGN.md §9k: evaluate.py for stage2.pth and for a checkpoint fine-tuned on random layouts
(--policy), on random scenarios with K in {8, 16, 32} robots (default 10 m square, 1024 worlds, one episode per robot,
the §9i runs), on the 50-robot circle (8 worlds, one episode) and on stage 2 (8 worlds, 3 episodes; the §9c runs),
seed 0.  Prints the card and power limit, then one markdown row per run.

    python tools/random_train_table.py --policy policy/stage2_600.pth
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

RUNS = [('random K = %d' % K, ['--scenario', 'random', '--random-robots', str(K), '--num-worlds', '1024'])
        for K in (8, 16, 32)] + \
       [('circle', ['--scenario', 'circle', '--num-worlds', '8', '--episodes', '1']),
        ('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3'])]


def row(name, scenario, out):
    m = out['metrics']
    f = lambda key: '–' if m[key][0] != m[key][0] else '%.3f ± %.3f' % m[key]
    return '| %s | %s | %d | %d | %d | %.3f | %.3f | %.3f | %d | %s | %s | %s |' % (
        name, scenario, out['partials'].shape[0], out['ticks'], m['episodes'], m['success_rate'], m['crash_rate'],
        m['timeout_rate'], m['unfinished'], f('extra_time'), f('extra_distance'), f('average_speed'))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--policy', required=True, help='the fine-tuned checkpoint')
    ap.add_argument('--name', default=None, help='its name in the table (default: the file name)')
    args = ap.parse_args(argv)
    if not os.path.exists(args.policy):
        ap.error('policy file %s not found' % args.policy)
    controllers = [('`stage2.pth`', os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')),
                   (args.name or '`%s`' % os.path.basename(args.policy), args.policy)]
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    print('| controller | scenario | worlds | ticks | episodes | success | crash | time-out | unfinished | extra time | '
          'extra distance | average speed |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|')
    for scenario, run in RUNS:
        for name, path in controllers:
            with contextlib.redirect_stdout(io.StringIO()):
                out = evaluate.main(run + ['--seed', '0', '--policy', path])
            print(row(name, scenario, out), flush=True)
            del out
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
