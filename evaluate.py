#!/usr/bin/env python
"""Deterministic evaluation of a policy on stage 1, stage 2 or the circle swap, with the metrics of the paper the
reference accompanies (DESIGN.md §9c): success / crash / time-out rates, and over the successful episodes the mean and
population std of extra time, extra distance and average speed.  Every robot drives with the policy's mean action
(--policy), with the ORCA-DD baseline controller (--baseline orca, DESIGN.md §9d) or with the paper's NH-ORCA baseline
(--baseline nh-orca, DESIGN.md §9e) until it has --episodes recorded episodes (circle: one) or --max-ticks ticks have
run.  --orca-map lets either baseline see the static map's walls (obstacle half-planes, DESIGN.md §9f).

    python evaluate.py --scenario stage1 --policy tests/golden/checkpoints/stage1_2.pth --num-worlds 8 --episodes 3
    python evaluate.py --scenario circle --policy tests/golden/checkpoints/stage2.pth --num-worlds 2 --episodes 1 \\
        --circle-robots 24 --circle-radius 12 --json circle.json
    python evaluate.py --scenario stage2 --baseline orca --num-worlds 8 --episodes 3
    python evaluate.py --scenario stage2 --baseline nh-orca --num-worlds 8 --episodes 3
    python evaluate.py --scenario stage2 --baseline nh-orca --orca-map --num-worlds 8 --episodes 3
"""
import argparse
import json
import os

import torch

from rl_collision_avoidance_b200.evaluation import AUTO_RESET, COLUMNS, evaluate
from rl_collision_avoidance_b200.model.net import CNNPolicy
from rl_collision_avoidance_b200.orca import DEFAULTS as ORCA_DEFAULTS, NH_DEFAULTS, OBSTACLE_TIME_HORIZON, \
    NhOrcaController, OrcaController
from rl_collision_avoidance_b200.scenarios import make_scenario
from rl_collision_avoidance_b200.stage_world import StageWorld

LASER_BEAM = 512
LASER_HIST = 3
CIRCLE_MAX_TICKS = 1500          # 25 m radius: the 49.5 m to the goal radius take at least 495 ticks at v_max


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--scenario', required=True, choices=sorted(AUTO_RESET))
    who = ap.add_mutually_exclusive_group(required=True)
    who.add_argument('--policy', help='state_dict of CNNPolicy (e.g. tests/golden/checkpoints/stage2.pth)')
    who.add_argument('--baseline', choices=['orca', 'nh-orca'],
                     help='drive with the ORCA-DD or the NH-ORCA controller instead of a policy')
    ap.add_argument('--orca-radius', type=float, default=None,
                    help='robot radius, m (default %g for orca, %g for nh-orca)'
                    % (ORCA_DEFAULTS['radius'], NH_DEFAULTS['radius']))
    ap.add_argument('--orca-horizon', type=float, default=ORCA_DEFAULTS['time_horizon'], help='time horizon tau, s')
    ap.add_argument('--orca-neighbour-dist', type=float, default=ORCA_DEFAULTS['neighbour_dist'],
                    help='neighbours are the robots closer than this, m')
    ap.add_argument('--orca-gain', type=float, default=None,
                    help='ORCA-DD heading gain k_w, 1/s (default %g)' % ORCA_DEFAULTS['heading_gain'])
    ap.add_argument('--nh-error', type=float, default=NH_DEFAULTS['tracking_error'],
                    help='NH-ORCA tracking error E, m')
    ap.add_argument('--nh-heading-time', type=float, default=NH_DEFAULTS['heading_time'],
                    help='NH-ORCA heading time T, s')
    ap.add_argument('--orca-map', action='store_true',
                    help='the baseline also avoids the static map (obstacle half-planes from the occupancy grid)')
    ap.add_argument('--orca-obstacle-horizon', type=float, default=None,
                    help='obstacle time horizon tau_o, s, with --orca-map (default %g)' % OBSTACLE_TIME_HORIZON)
    ap.add_argument('--num-worlds', type=int, default=1)
    ap.add_argument('--episodes', type=int, default=1, help='recorded episodes per robot (circle: at most 1)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--max-ticks', type=int, default=None,
                    help='default: episodes x (timeout + 1) on stage 1 / 2, %d on the circle' % CIRCLE_MAX_TICKS)
    ap.add_argument('--circle-robots', type=int, default=None, help='K robots on the circle (default: the 50-row table)')
    ap.add_argument('--circle-radius', type=float, default=None, help='circle radius in metres (default 25)')
    ap.add_argument('--check-every', type=int, default=50)
    ap.add_argument('--json', default=None, help='write totals, metrics and per-world partials here')
    args = ap.parse_args(argv)
    if args.policy is not None and not os.path.exists(args.policy):
        ap.error('policy file %s not found' % args.policy)
    if args.baseline != 'orca' and args.orca_gain is not None:
        ap.error('--orca-gain applies to --baseline orca only')
    if args.baseline is None and args.orca_map:
        ap.error('--orca-map applies to --baseline orca / nh-orca only')
    if not args.orca_map and args.orca_obstacle_horizon is not None:
        ap.error('--orca-obstacle-horizon applies with --orca-map only')
    obstacle_horizon = OBSTACLE_TIME_HORIZON if args.orca_obstacle_horizon is None else args.orca_obstacle_horizon
    if args.scenario != 'circle' and (args.circle_robots is not None or args.circle_radius is not None):
        ap.error('--circle-robots / --circle-radius apply to --scenario circle only')
    sc = make_scenario(args.scenario, robots_per_world=args.circle_robots, radius=args.circle_radius) \
        if args.scenario == 'circle' else make_scenario(args.scenario)
    env = StageWorld(LASER_BEAM, index=0, scenario=sc, num_worlds=args.num_worlds, seed=args.seed,
                     auto_reset=AUTO_RESET[args.scenario])
    if args.baseline == 'orca':
        gain = ORCA_DEFAULTS['heading_gain'] if args.orca_gain is None else args.orca_gain
        radius = ORCA_DEFAULTS['radius'] if args.orca_radius is None else args.orca_radius
        policy = OrcaController(env, radius=radius, neighbour_dist=args.orca_neighbour_dist,
                                time_horizon=args.orca_horizon, heading_gain=gain, obstacles=args.orca_map,
                                obstacle_time_horizon=obstacle_horizon)
        controller = 'orca-dd+map' if args.orca_map else 'orca-dd'
    elif args.baseline == 'nh-orca':
        radius = NH_DEFAULTS['radius'] if args.orca_radius is None else args.orca_radius
        policy = NhOrcaController(env, radius=radius, neighbour_dist=args.orca_neighbour_dist,
                                  time_horizon=args.orca_horizon, tracking_error=args.nh_error,
                                  heading_time=args.nh_heading_time, obstacles=args.orca_map,
                                  obstacle_time_horizon=obstacle_horizon)
        controller = 'nh-orca+map' if args.orca_map else 'nh-orca'
    else:
        policy = CNNPolicy(frames=LASER_HIST, action_space=2, max_batch=env.N)
        policy.load_state_dict(torch.load(args.policy, map_location='cuda'))
        controller = None
    max_ticks = args.max_ticks if args.max_ticks is not None else \
        (CIRCLE_MAX_TICKS if args.scenario == 'circle' else args.episodes * (sc.timeout + 1))
    out = evaluate(env, policy, args.episodes, max_ticks, check_every=args.check_every)
    m = out['metrics']
    f = lambda k: '%.3f +- %.3f' % m[k]
    print(('%s  ' % controller if controller else '') +
          '%s  robots %d  ticks %d  episodes %d  success %.4f  crash %.4f  time-out %.4f  unfinished %d  '
          'extra time %s s  extra distance %s m  average speed %s m/s'
          % (args.scenario, env.N, out['ticks'], m['episodes'], m['success_rate'], m['crash_rate'], m['timeout_rate'],
             m['unfinished'], f('extra_time'), f('extra_distance'), f('average_speed')))
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump({'args': vars(args), 'controller': controller or 'policy', 'robots': env.N,
                       'ticks': out['ticks'], 'metrics': m,
                       'columns': list(COLUMNS), 'totals': out['totals'].tolist(),
                       'partials': out['partials'].tolist()}, fh, indent=1)
    return out


if __name__ == '__main__':
    main()
