#!/usr/bin/env python
"""The results of DESIGN.md §9z: fine-tunes of `stage2.pth` on arenas (arena seed 0, 256 worlds x 8 robots, 100
updates) in two arms, uniform arena draws (pick 1) and --arena-curriculum (default parameters), with training seeds 0,
1 and 2 in each.  Every checkpoint is evaluated with evaluate.py --timeouts on held-out arena seed 1 (64 worlds) and
on stage 2 (8 worlds, 2 episodes per robot), and with --per-arena on the training arenas (seed 0, 64 worlds: one per
arena).  Each fine-tune runs ppo_stage2.py in its own temporary directory.  Prints the card, power limit and maximum
SM clock, each fine-tune's last training lines, one markdown row per fine-tune and the mean of each arm.  Three seeds
per arm: observations, not effect sizes.

    python tools/curriculum_table.py [--updates 100] [--seeds 0,1,2]
"""
import argparse
import contextlib
import io
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import evaluate  # noqa: E402
from rl_collision_avoidance_b200.evaluation import per_arena  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402

STAGE2 = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')
ARMS = [('uniform', []), ('curriculum', ['--arena-curriculum'])]
HELD_OUT = ['--scenario', 'arena', '--arena-robots', '8', '--num-worlds', '64', '--arena-seed', '1', '--timeouts']
STAGE_2 = ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '2', '--timeouts']
TRAINING = ['--scenario', 'arena', '--arena-robots', '8', '--num-worlds', '64', '--arena-seed', '0', '--per-arena']


def fine_tune(d, flags, updates, seed):
    """ppo_stage2.py in directory d from stage2.pth; returns the last checkpoint, the output's last lines and the
    curriculum's final effective arena count (None without one)."""
    os.makedirs(os.path.join(d, 'policy'))
    shutil.copy(STAGE2, os.path.join(d, 'policy', 'stage2.pth'))
    cmd = [sys.executable, os.path.join(ROOT, 'ppo_stage2.py'), '--scenario', 'arena', '--arena-robots', '8',
           '--arena-seed', '0', '--num-worlds', '256', '--updates', str(updates), '--seed', str(seed)] + flags
    out = subprocess.run(cmd, cwd=d, capture_output=True, text=True, check=True).stdout
    tail = [l for l in out.splitlines() if l.startswith(('update ', 'last update'))]
    m = re.search(r'curriculum: \d+ arenas, effective ([0-9.]+)', out)
    return os.path.join(d, 'policy', 'stage2_%d.pth' % updates), tail, float(m.group(1)) if m else None


def _eval(argv):
    with contextlib.redirect_stdout(io.StringIO()):
        return evaluate.main(argv + ['--seed', '0'])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--updates', type=int, default=100, help='fine-tune updates (a multiple of 20: the checkpoint step)')
    ap.add_argument('--seeds', default='0,1,2')
    args = ap.parse_args()
    seeds = [int(s) for s in args.seeds.split(',')]
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info), flush=True)
    rows = {}
    for arm, flags in ARMS:
        for seed in seeds:
            with tempfile.TemporaryDirectory() as d:
                ckpt, tail, eff = fine_tune(d, flags, args.updates, seed)
                print('fine-tune %s seed %d: %s' % (arm, seed, ' | '.join(tail)), flush=True)
                held, st2 = _eval(HELD_OUT + ['--policy', ckpt])['metrics'], _eval(STAGE_2 + ['--policy', ckpt])['metrics']
                tr = _eval(TRAINING + ['--policy', ckpt])
                lay = make_scenario('arena', robots_per_world=8, arena_seed=0).layout
                succ = [r['metrics']['success_rate'] for r in per_arena(tr['partials'], lay)
                        if r['metrics']['episodes']]
                v = [held['success_rate'], held['crash_rate'], held['timeout_rate'], held['unfinished'],
                     st2['success_rate'], st2['crash_rate'], tr['metrics']['success_rate'], float(np.min(succ)),
                     float(np.mean(np.asarray(succ) < 0.75)), eff if eff is not None else float('nan')]
                rows.setdefault(arm, []).append(v)
                print(_row('%s, seed %d' % (arm, seed), v), flush=True)
    print('| fine-tune | held-out success | crash | time-out | unfinished | stage 2 success | crash | training '
          'arenas success | lowest arena | arenas < 0.75 | effective arenas |')
    print('|---|---|---|---|---|---|---|---|---|---|---|')
    for arm, _ in ARMS:
        for seed, v in zip(seeds, rows[arm]):
            print(_row('%s, seed %d' % (arm, seed), v))
        print(_row('%s, mean of %d' % (arm, len(seeds)), list(np.mean(rows[arm], 0))))


def _row(name, v):
    return ('| %s | %.4f | %.4f | %.4f | %.1f | %.4f | %.4f | %.4f | %.3f | %.3f | %.1f |' % (name, *v))


if __name__ == '__main__':
    main()
