#!/usr/bin/env python
"""The results of DESIGN.md §9u: evaluate.py --timeouts for stage2.pth, NH-ORCA+map and the dynamic-window baseline on
stage 2 (8 worlds, --episodes 3), the 50-robot circle (8 worlds) and random layouts (K = 16 robots, 64 worlds), seed 0,
clean and under scan noise (--scan-noise 0.05 --beam-dropout 0.1), scan delay (--scan-delay 2) and localization error
(--pose-error 0.1,0.3).  NH-ORCA reads the true state, so the sensing conditions do not apply to it.  Prints one
markdown row per run (time-outs and unfinished episodes split into frozen / stalled / slow, and DWA's fallback share),
and the card and power limit.

    python tools/dwa_table.py
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
               ('DWA', ['--baseline', 'dwa'])]
SCENARIOS = [('stage 2', ['--scenario', 'stage2', '--num-worlds', '8', '--episodes', '3']),
             ('circle', ['--scenario', 'circle', '--num-worlds', '8']),
             ('random K = 16', ['--scenario', 'random', '--random-robots', '16', '--num-worlds', '64'])]
CONDITIONS = [('clean', []), ('scan noise 0.05, dropout 0.1', ['--scan-noise', '0.05', '--beam-dropout', '0.1']),
              ('scan delay 2', ['--scan-delay', '2']), ('pose error 0.1..0.3', ['--pose-error', '0.1,0.3'])]


def row(name, scenario, condition, out):
    m, p = out['metrics'], out['progress']
    f = lambda key: '–' if m[key][0] != m[key][0] else '%.3f ± %.3f' % m[key]
    stuck = lambda g: '%d / %d / %d' % (p[g + '_frozen'], p[g + '_stalled'], p[g + '_slow'])
    fb = '%.4f' % out['dwa']['fallback_share'] if 'dwa' in out else '–'
    return '| %s | %s | %s | %d | %.3f | %.3f | %.3f | %d | %s | %s | %s | %s |' % (
        name, scenario, condition, m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
        m['unfinished'], stuck('timeout'), stuck('unfinished'), f('extra_time'), fb)


def main():
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    print('| controller | scenario | condition | episodes | success | crash | time-out | unfinished | '
          'time-outs frozen / stalled / slow | unfinished frozen / stalled / slow | extra time | DWA fallback |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|')
    for sname, sargv in SCENARIOS:
        for cname, cargv in CONDITIONS:
            for name, who in CONTROLLERS:
                if cargv and name.startswith('NH-ORCA'):
                    continue
                with contextlib.redirect_stdout(io.StringIO()):
                    out = evaluate.main(sargv + who + cargv + ['--timeouts', '--seed', '0'])
                print(row(name, sname, cname, out), flush=True)


if __name__ == '__main__':
    main()
