#!/usr/bin/env python
"""The results of DESIGN.md §9x: three fine-tunes of `stage2.pth` on arenas (arena seed 0, 256 worlds x 8 robots, 100
updates, seed 0) - no planner, `--planner --planner-reward straight` and `--planner` - each evaluated with
evaluate.py --timeouts on held-out arena seed 1 (64 worlds) and on stage 2 (8 worlds, 2 episodes per robot), with
--geodesic and with --planner, in tools/planner_table.py's columns.  Each fine-tune runs ppo_stage2.py in its own
temporary directory (its policy/ and log/ stay there).  Prints the card, power limit and maximum SM clock, each
fine-tune's last training line and one markdown row per evaluation.  One seed: observations, not effect sizes.

    python tools/planner_train_table.py [--updates 100]
"""
import argparse
import contextlib
import io
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import evaluate  # noqa: E402
from planner_table import row  # noqa: E402

STAGE2 = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')
ARMS = [('no planner', []), ('straight', ['--planner', '--planner-reward', 'straight']), ('geodesic', ['--planner'])]
SCENARIOS = [('arenas, seed 1', ['--scenario', 'arena', '--arena-robots', '8', '--num-worlds', '64',
                                 '--arena-seed', '1']),
             ('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '2'])]


def fine_tune(d, flags, updates):
    """ppo_stage2.py in directory d from stage2.pth; returns the checkpoint of the last update and the output's last
    lines."""
    os.makedirs(os.path.join(d, 'policy'))
    shutil.copy(STAGE2, os.path.join(d, 'policy', 'stage2.pth'))
    cmd = [sys.executable, os.path.join(ROOT, 'ppo_stage2.py'), '--scenario', 'arena', '--arena-robots', '8',
           '--arena-seed', '0', '--num-worlds', '256', '--updates', str(updates), '--seed', '0'] + flags
    out = subprocess.run(cmd, cwd=d, capture_output=True, text=True, check=True).stdout
    tail = [l for l in out.splitlines() if l.startswith(('update ', 'last update'))]
    return os.path.join(d, 'policy', 'stage2_%d.pth' % updates), tail


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--updates', type=int, default=100, help='fine-tune updates (a multiple of 20: the checkpoint step)')
    args = ap.parse_args()
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info), flush=True)
    rows = []
    for arm, flags in ARMS:
        with tempfile.TemporaryDirectory() as d:
            ckpt, tail = fine_tune(d, flags, args.updates)
            print('fine-tune %s: %s' % (arm, ' | '.join(tail)), flush=True)
            for sname, sargv in SCENARIOS:
                for steer in ('--geodesic', '--planner'):
                    with contextlib.redirect_stdout(io.StringIO()):
                        out = evaluate.main(sargv + ['--policy', ckpt, steer, '--timeouts', '--seed', '0'])
                    name = '%s%s' % (arm, ' + planner' if steer == '--planner' else '')
                    rows.append(row(name, sname, out))
                    print(rows[-1], flush=True)
    print('| fine-tune | scenario | episodes | success | crash | time-out | unfinished (frozen / stalled / slow) | '
          'extra distance m | extra geodesic distance m | goal visible / waypoint / no plan | no path |')
    print('|---|---|---|---|---|---|---|---|---|---|---|')
    for r in rows:
        print(r)


if __name__ == '__main__':
    main()
