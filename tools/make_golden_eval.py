#!/usr/bin/env python
"""Record the per-world partials of evaluate() on the checkpoint and baseline runs the evaluation tests use (DESIGN.md
§9c), so that later changes to the evaluation loop can be checked bit for bit against them.  Needs a GPU.

    python tools/make_golden_eval.py --out tests/golden/eval_partials.npz
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CKPT = os.path.join(ROOT, 'tests', 'golden', 'checkpoints')

# name: (scenario, worlds, seed, controller: checkpoint file or 'orca' / 'nh-orca', episodes, max_ticks, check_every)
RUNS = {
    'stage1_policy': ('stage1', 2, 3, 'stage1_2.pth', 3, 300, 25),
    'stage2_policy': ('stage2', 3, 2, 'stage2.pth', 2, 402, 50),
    'circle_policy': ('circle', 2, 4, 'stage2.pth', 1, 50, 50),
    'circle_orca': ('circle', 2, 4, 'orca', 1, 200, 50),
    'stage2_nh_orca_map': ('stage2', 3, 2, 'nh-orca', 2, 402, 50),
}


def run(name):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET, evaluate
    from rl_collision_avoidance_b200.model.net import CNNPolicy
    from rl_collision_avoidance_b200.orca import NhOrcaController, OrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    scenario, worlds, seed, who, episodes, max_ticks, check_every = RUNS[name]
    env = StageWorld(512, scenario=scenario, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[scenario])
    if who == 'orca':
        policy = OrcaController(env)
    elif who == 'nh-orca':
        policy = NhOrcaController(env, obstacles=True)
    else:
        policy = CNNPolicy(frames=3, action_space=2, max_batch=env.N)
        policy.load_state_dict(torch.load(os.path.join(CKPT, who), map_location='cpu'))
    out = evaluate(env, policy, episodes, max_ticks, check_every=check_every)
    return out['partials'], out['ticks']


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--out', required=True)
    args = ap.parse_args()
    arrays = {}
    for name in RUNS:
        partials, ticks = run(name)
        arrays['partials_' + name] = partials
        arrays['ticks_' + name] = np.int64(ticks)
        print(name, ticks, partials.sum(0)[:4], flush=True)
    np.savez(args.out, **arrays)


if __name__ == '__main__':
    main()
