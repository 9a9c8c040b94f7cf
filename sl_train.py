#!/usr/bin/env python
"""Train the paper's SL-policy baseline (DESIGN.md §9g): the CNNPolicy network fitted by behaviour cloning to the
actions of a baseline controller (NH-ORCA with the map by default), recorded on the device while the controller drives
each --scenario for --samples rows.  --holdout of the rows is kept out of training; every epoch prints the training loss
(the mean of its minibatch losses) and the held-out loss.  The checkpoint is a CNNPolicy state_dict that
`evaluate.py --policy` loads.

    python sl_train.py --out sl_policy.pth
    python sl_train.py --scenario stage1 --samples 8000 --epochs 2 --out /tmp/sl.pth
    python evaluate.py --scenario stage2 --policy sl_policy.pth --num-worlds 8 --episodes 3

The defaults (2 x 400 000 rows, batch 1024, the learning rate and epoch count below) are starting values, not tuned
ones: the learning rate and the epoch count were picked from one sweep of held-out losses on an H100 (DESIGN.md §9g).
"""
import argparse
import math
import os
import time

import torch

from rl_collision_avoidance_b200.evaluation import AUTO_RESET
from rl_collision_avoidance_b200.orca import add_arguments as add_controller_arguments, \
    check_arguments as check_controller_arguments, from_arguments as controller_from_arguments

LASER_BEAM = 512
LASER_HIST = 3
DEFAULT_SCENARIOS = ['stage1', 'stage2']
DEFAULT_LR = 3e-4
DEFAULT_EPOCHS = 11


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--scenario', action='append', choices=sorted(AUTO_RESET), default=None,
                    help='record on this scenario (repeatable; default: %s)' % ' + '.join(DEFAULT_SCENARIOS))
    ap.add_argument('--samples', type=int, default=400000, help='rows recorded per scenario')
    ap.add_argument('--baseline', choices=['orca', 'nh-orca'], default='nh-orca', help='the expert controller')
    add_controller_arguments(ap, map_default=True)
    ap.add_argument('--num-worlds', type=int, default=16)
    ap.add_argument('--record-every', type=int, default=1, help='record every k-th tick')
    ap.add_argument('--epochs', type=int, default=DEFAULT_EPOCHS)
    ap.add_argument('--batch-size', type=int, default=1024)
    ap.add_argument('--lr', type=float, default=DEFAULT_LR, help='Adam learning rate')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--holdout', type=float, default=0.05, help='fraction of the rows kept out of training')
    ap.add_argument('--out', required=True, help='where to write the CNNPolicy state_dict')
    args = ap.parse_args(argv)
    check_controller_arguments(ap, args)
    if args.scenario is None:
        args.scenario = list(DEFAULT_SCENARIOS)
    for name in ('samples', 'num_worlds', 'record_every', 'epochs', 'batch_size'):
        if getattr(args, name) < 1:
            ap.error('--%s must be >= 1' % name.replace('_', '-'))
    if not (math.isfinite(args.lr) and args.lr > 0):
        ap.error('--lr must be finite and > 0')
    if not 0 <= args.holdout < 1:
        ap.error('--holdout must be in [0, 1)')
    out_dir = os.path.dirname(os.path.abspath(args.out))
    if not os.path.isdir(out_dir):
        ap.error('the directory of --out (%s) does not exist' % out_dir)
    return args


def main(argv=None):
    args = parse(argv)
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.sl import collect, sl_loss, sl_update
    from rl_collision_avoidance_b200.stage_world import StageWorld
    parts = []
    for name in args.scenario:
        t0 = time.time()
        env = StageWorld(LASER_BEAM, index=0, scenario=name, num_worlds=args.num_worlds, seed=args.seed,
                         auto_reset=AUTO_RESET[name])
        ctrl, label = controller_from_arguments(env, args)
        data = collect(env, ctrl, args.samples, record_every=args.record_every)
        torch.cuda.synchronize()
        print('%s  %s  robots %d  rows %d  (%.1f s)' % (name, label, env.N, data[0].shape[0], time.time() - t0),
              flush=True)
        parts.append(data)
        del env, ctrl
    data = tuple(torch.cat([p[i] for p in parts]) for i in range(3))
    del parts
    n = data[0].shape[0]
    split = torch.Generator(device='cpu')
    split.manual_seed(args.seed)
    perm = torch.randperm(n, generator=split).to(data[0].device)
    n_hold = int(round(args.holdout * n))
    held, train = perm[:n_hold], perm[n_hold:]
    if train.numel() < 1:
        raise SystemExit('no training rows: record more samples or lower --holdout')
    policy = CNNPolicy(frames=LASER_HIST, action_space=2, seed=args.seed, max_batch=args.batch_size)
    opt = Adam(policy.parameters(), lr=args.lr)
    gen = torch.Generator(device=policy.device)
    gen.manual_seed(args.seed)
    held_loss = lambda: sl_loss(policy, data, args.batch_size, rows=held) if n_hold else math.nan
    print('rows %d  train %d  held-out %d  batch %d  lr %g' % (n, train.numel(), n_hold, args.batch_size, args.lr))
    print('epoch 0  held-out loss %.6f' % held_loss(), flush=True)
    for epoch in range(1, args.epochs + 1):
        t0 = time.time()
        losses = sl_update(policy, opt, data, args.batch_size, 1, generator=gen, rows=train)
        print('epoch %d  train loss %.6f  held-out loss %.6f  (%.1f s)'
              % (epoch, sum(losses) / len(losses), held_loss(), time.time() - t0), flush=True)
    torch.save({k: v.cpu() for k, v in policy.state_dict().items()}, args.out)
    print('wrote %s' % args.out)
    return policy


if __name__ == '__main__':
    main()
