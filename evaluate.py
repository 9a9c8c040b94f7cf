#!/usr/bin/env python
"""Deterministic evaluation of a policy on stage 1, stage 2, the circle swap, random or arena scenarios, with the metrics of
the paper the reference accompanies (DESIGN.md §9c): success / crash / time-out rates, and over the successful episodes
the mean and population std of extra time, extra distance and average speed.  Every robot drives with the policy's
mean action (--policy), with the ORCA-DD baseline controller (--baseline orca, DESIGN.md §9d) or with the paper's
NH-ORCA baseline (--baseline nh-orca, DESIGN.md §9e) until it has --episodes recorded episodes (circle and random: one)
or --max-ticks ticks have run.  --orca-map lets either baseline see the static map's walls (obstacle half-planes,
DESIGN.md §9f).  --non-cooperative K makes K robots of every world drive straight to their goals, ignoring everyone else, and adds the
metrics of each role (DESIGN.md §9h).  --scenario random gives every world its own layout: --random-robots K robots
start at random positions in a --random-side S m square on circle.world's map, at least --random-separation D m apart,
with random goals at least --random-min-travel L m away (defaults 8, 10, 1 and S / 2; DESIGN.md §9i).  --scenario arena
does the same among static obstacles: world w lays out in arena w mod T of a generated map of --arena-count T walled
arenas of --arena-side S m with --arena-obstacles LO,HI random boxes and discs each, drawn from --arena-seed (another
seed gives held-out arenas), with --arena-robots, --arena-separation and --arena-min-travel (defaults 64, 10, 4,10, 0,
8, 1.2 and S / 2; DESIGN.md §9v); --per-arena adds each arena's episodes and rates to --json and prints the ten arenas
of lowest success (DESIGN.md §9z).  --hybrid switches
the policy per robot by the nearest return of its newest scan: straight to the goal when it is beyond
--hybrid-r-safe, the policy's action with v capped at --hybrid-v-safe when it is within --hybrid-r-risk, the policy's
action otherwise, and prints the share of robot-ticks in each mode (DESIGN.md §9j).  --safety adds how closely the robots
passed and why they crashed: crashes by cause (static map / another robot), and over the successful episodes the
minimum separation between footprints, the minimum clearance and the near-miss rate, a near miss being a tick closer
than --near-miss D m (default 0.1) to another robot (DESIGN.md §9m).  --timeouts adds why robots timed out or never
finished: each time-out and each unfinished episode is called frozen (its centre has not moved for --stall-window W
ticks, default 50), stalled (it moves but has not come 0.1 m closer to its goal in W ticks) or slow (still getting
closer), and marked when another robot stood within 1 m; with the closest distance to the goal left, the share of
still ticks and the rotation per successful episode (DESIGN.md §9o).  --scan-noise SIGMA_M, --beam-dropout P and
--action-noise SIGMA_V[,SIGMA_W] evaluate under sensor and actuation noise: Gaussian range error on every beam with a
return, beams that read no return, and a relative gain error on the executed v and w, drawn from --noise-seed
(default --seed; DESIGN.md §9p).  The ORCA baselines do not read the scan, so only --action-noise applies to them.
--scan-delay T[,T_MAX] and --command-delay T[,T_MAX] evaluate under sensing and command latency: each robot reads the
scan of T ticks (0.1 s each) earlier and executes the command issued T ticks earlier, or a delay drawn in T..T_MAX per
robot and episode from --latency-seed (default --seed; DESIGN.md §9q).  Only --command-delay applies to the baselines.
--accel-limit A[,A_MAX] and --angular-accel-limit B[,B_MAX] evaluate under acceleration limits: each tick the executed v
changes by at most A dt and w by at most B dt, with limits drawn in A..A_MAX and B..B_MAX per robot and episode from
--dynamics-seed (default --seed; DESIGN.md §9r).  They apply to the baselines too.
--pose-error S[,S_MAX], --heading-error S[,S_MAX] and --speed-error SV[,SW] evaluate under localization error: the
policy's local goal is computed from a believed pose whose position and heading errors have standard deviations S m and
S rad (or drawn in S..S_MAX per robot and episode) and a correlation time of --pose-error-time T s (default 2; 0 new on
every tick, inf one offset per episode), and the speed it reads carries white noise, from --localization-seed (default
--seed; DESIGN.md §9s).  Success, crashes and every metric stay on the true poses.  --policy only, not --hybrid.
--crowd K makes K agents of every world a social-force crowd that avoids each other, the other agents (not with
--crowd-ignores-robots) and, with --crowd-map, the static map, with --crowd-speed, --crowd-strength, --crowd-range and
--crowd-side-bias; the metrics are also printed per role (DESIGN.md §9t).  Not with --non-cooperative.
--baseline dwa drives every robot with the dynamic-window baseline, which reads what the policy reads (the newest scan,
the local goal and its speed), so every sensing perturbation applies to it; --dwa-radius, --dwa-horizon,
--dwa-heading-time, --dwa-samples V,W, --dwa-accel A[,B], --dwa-brake and --dwa-weights H,C,S set it (DESIGN.md §9u).
--planner steers the policy (or --baseline dwa) by a global planner on the device: where a robot's goal is out of sight
its local goal is the farthest visible cell of the geodesic path; it prints the share of robot-ticks that saw the goal,
followed a waypoint or had no plan, and the geodesic metrics.  --geodesic prints only the geodesic metrics (the
geodesic length of every episode and the extra geodesic distance), for any controller (DESIGN.md §9w).  Neither works
on a map too big to plan on (circle.world).

    python evaluate.py --scenario stage1 --policy tests/golden/checkpoints/stage1_2.pth --num-worlds 8 --episodes 3
    python evaluate.py --scenario circle --policy tests/golden/checkpoints/stage2.pth --num-worlds 2 --episodes 1 \\
        --circle-robots 24 --circle-radius 12 --json circle.json
    python evaluate.py --scenario stage2 --baseline orca --num-worlds 8 --episodes 3
    python evaluate.py --scenario stage2 --baseline nh-orca --num-worlds 8 --episodes 3
    python evaluate.py --scenario stage2 --baseline nh-orca --orca-map --num-worlds 8 --episodes 3
    python evaluate.py --scenario circle --policy tests/golden/checkpoints/stage2.pth --num-worlds 8 --episodes 1 \\
        --non-cooperative 5
    python evaluate.py --scenario random --baseline nh-orca --orca-map --num-worlds 1024 --random-robots 16
    python evaluate.py --scenario random --policy tests/golden/checkpoints/stage2.pth --num-worlds 1024 --hybrid
    python evaluate.py --scenario arena --baseline nh-orca --orca-map --num-worlds 64 --arena-seed 1
    python evaluate.py --scenario stage2 --policy tests/golden/checkpoints/stage2.pth --num-worlds 8 --episodes 3 --safety
    python evaluate.py --scenario stage2 --policy tests/golden/checkpoints/stage1_2.pth --num-worlds 8 --episodes 3 \\
        --timeouts
    python evaluate.py --scenario stage2 --policy tests/golden/checkpoints/stage2.pth --num-worlds 8 --episodes 3 \\
        --scan-noise 0.05 --beam-dropout 0.1 --action-noise 0.1
    python evaluate.py --scenario stage2 --policy tests/golden/checkpoints/stage2.pth --num-worlds 8 --episodes 3 \\
        --scan-delay 2 --command-delay 1,3
    python evaluate.py --scenario stage2 --policy tests/golden/checkpoints/stage2.pth --num-worlds 8 --episodes 3 \\
        --accel-limit 1 --angular-accel-limit 2
    python evaluate.py --scenario stage2 --policy tests/golden/checkpoints/stage2.pth --num-worlds 8 --episodes 3 \\
        --pose-error 0.1,0.3 --heading-error 0.05 --speed-error 0.05,0.1
    python evaluate.py --scenario stage2 --policy tests/golden/checkpoints/stage2.pth --num-worlds 8 --episodes 3 \\
        --crowd 5 --crowd-map
    python evaluate.py --scenario stage2 --baseline dwa --num-worlds 8 --episodes 3 --scan-noise 0.05 --timeouts
"""
import argparse
import json
import math
import os

import torch

from rl_collision_avoidance_b200.crowd import CROWD_FLAGS, Crowd, add_crowd_arguments, crowd_from_arguments
from rl_collision_avoidance_b200.dwa import DWA_FLAGS, DwaController, add_arguments as add_dwa_arguments, \
    check_arguments as check_dwa_arguments, from_arguments as dwa_from_arguments
from rl_collision_avoidance_b200.dynamics import DYNAMICS_FLAGS, Dynamics, add_dynamics_arguments, \
    dynamics_from_arguments
from rl_collision_avoidance_b200.evaluation import AUTO_RESET, COLUMNS, PROGRESS_COLUMNS, PROGRESS_DEFAULTS, \
    SAFETY_COLUMNS, evaluate, non_cooperative_mask, per_arena
from rl_collision_avoidance_b200.latency import LATENCY_FLAGS, Latency, add_latency_arguments, \
    latency_from_arguments
from rl_collision_avoidance_b200.localization import LOCALIZATION_FLAGS, Localization, add_localization_arguments, \
    localization_from_arguments
from rl_collision_avoidance_b200.model.net import CNNPolicy
from rl_collision_avoidance_b200.planner import PARTIALS as GEODESIC_COLUMNS, Planner, \
    add_arguments as add_planner_arguments, build_plan_tables, check_arguments as check_planner_arguments, \
    from_arguments as planner_from_arguments
from rl_collision_avoidance_b200.noise import NOISE_FLAGS, Noise, add_noise_arguments, noise_from_arguments
from rl_collision_avoidance_b200.orca import HYBRID_DEFAULTS, Hybrid, NonCooperative, \
    add_arguments as add_controller_arguments, check_arguments as check_controller_arguments, check_hybrid, \
    from_arguments as controller_from_arguments
from rl_collision_avoidance_b200.scenarios import COMMON, add_arena_arguments, add_random_arguments, \
    arena_scenario_from_arguments, check_arena_arguments, check_random_arguments, make_scenario, random_max_ticks, \
    random_scenario_from_arguments
from rl_collision_avoidance_b200.stage_world import StageWorld

LASER_BEAM = 512
LASER_HIST = 3
CIRCLE_MAX_TICKS = 1500          # 25 m radius: the 49.5 m to the goal radius take at least 495 ticks at v_max


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--scenario', required=True, choices=sorted(AUTO_RESET))
    who = ap.add_mutually_exclusive_group(required=True)
    who.add_argument('--policy', help='state_dict of CNNPolicy (e.g. tests/golden/checkpoints/stage2.pth)')
    who.add_argument('--baseline', choices=['orca', 'nh-orca', 'dwa'],
                     help='drive with the ORCA-DD, the NH-ORCA or the dynamic-window controller instead of a policy')
    add_controller_arguments(ap)
    add_dwa_arguments(ap)
    ap.add_argument('--num-worlds', type=int, default=1)
    ap.add_argument('--episodes', type=int, default=1,
                    help='recorded episodes per robot (circle, random, arena: at most 1)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--max-ticks', type=int, default=None,
                    help='default: episodes x (timeout + 1) on stage 1 / 2, %d on the circle, '
                         '3 ceil(S sqrt(2) / (v_max dt)) on random and arena' % CIRCLE_MAX_TICKS)
    ap.add_argument('--circle-robots', type=int, default=None, help='K robots on the circle (default: the 50-row table)')
    ap.add_argument('--circle-radius', type=float, default=None, help='circle radius in metres (default 25)')
    add_random_arguments(ap)
    add_arena_arguments(ap)
    ap.add_argument('--check-every', type=int, default=50)
    ap.add_argument('--non-cooperative', type=int, default=None, metavar='K',
                    help='K robots per world (robots floor(j R / K), j < K) drive straight to their goals and ignore '
                         'everyone else; the metrics are also printed per role (DESIGN.md §9h)')
    ap.add_argument('--non-cooperative-speed', type=float, default=None, metavar='S',
                    help='speed of the non-cooperative robots, m/s, in (0, v_max] (default v_max)')
    add_crowd_arguments(ap)
    ap.add_argument('--hybrid', action='store_true',
                    help='switch the policy per robot by its nearest scan return: drive straight to the goal in free '
                         'space, cap the speed near obstacles (DESIGN.md §9j)')
    ap.add_argument('--hybrid-r-safe', type=float, default=None, metavar='R',
                    help='hybrid: drive straight to the goal when nothing is within R m (default %g)'
                         % HYBRID_DEFAULTS['r_safe'])
    ap.add_argument('--hybrid-r-risk', type=float, default=None, metavar='R',
                    help='hybrid: cap the speed when something is within R m (default %g)' % HYBRID_DEFAULTS['r_risk'])
    ap.add_argument('--hybrid-v-safe', type=float, default=None, metavar='V',
                    help='hybrid: the capped speed, m/s (default %g)' % HYBRID_DEFAULTS['v_safe'])
    ap.add_argument('--safety', action='store_true',
                    help='also report crashes by cause, minimum separation, minimum clearance and near misses '
                         '(DESIGN.md §9m)')
    ap.add_argument('--near-miss', type=float, default=None, metavar='D',
                    help='a tick closer than D m to another robot is a near miss (default 0.1); implies --safety')
    ap.add_argument('--timeouts', action='store_true',
                    help='also report why robots timed out or never finished: frozen, stalled or slow, with a robot '
                         'near or not (DESIGN.md §9o)')
    ap.add_argument('--stall-window', type=int, default=None, metavar='W',
                    help='a robot still for W ticks is frozen, one without progress for W ticks stalled (default %d); '
                         'implies --timeouts' % PROGRESS_DEFAULTS['window'])
    add_noise_arguments(ap)
    add_latency_arguments(ap)
    add_dynamics_arguments(ap)
    add_localization_arguments(ap)
    add_planner_arguments(ap)
    ap.add_argument('--per-arena', action='store_true',
                    help='arena scenario: metrics per arena (world w in arena w mod T) in --json, and the ten arenas '
                         'of lowest success printed (DESIGN.md §9z)')
    ap.add_argument('--json', default=None, help='write totals, metrics and per-world partials here')
    args = ap.parse_args(argv)
    if args.policy is not None and not os.path.exists(args.policy):
        ap.error('policy file %s not found' % args.policy)
    check_dwa_arguments(ap, args)
    check_controller_arguments(ap, args)
    orca = args.baseline in ('orca', 'nh-orca')
    if not orca and args.orca_map:
        ap.error('--orca-map applies to --baseline orca / nh-orca only')
    if args.scenario != 'circle' and (args.circle_robots is not None or args.circle_radius is not None):
        ap.error('--circle-robots / --circle-radius apply to --scenario circle only')
    check_arena_arguments(ap, args)
    check_random_arguments(ap, args)
    if args.per_arena and args.scenario != 'arena':
        ap.error('--per-arena applies to --scenario arena only')
    if args.non_cooperative is None and args.non_cooperative_speed is not None:
        ap.error('--non-cooperative-speed applies with --non-cooperative only')
    v_max = COMMON['v_max']
    if args.non_cooperative_speed is not None and not 0.0 < args.non_cooperative_speed <= v_max:
        ap.error('--non-cooperative-speed must be in (0, %g]' % v_max)
    hybrid_args = (args.hybrid_r_safe, args.hybrid_r_risk, args.hybrid_v_safe)
    if not args.hybrid and any(a is not None for a in hybrid_args):
        ap.error('--hybrid-r-safe / --hybrid-r-risk / --hybrid-v-safe apply with --hybrid only')
    if args.hybrid and args.baseline is not None:
        ap.error('--hybrid applies to --policy only')
    if args.near_miss is not None and not (math.isfinite(args.near_miss) and args.near_miss >= 0.0):
        ap.error('--near-miss must be finite and >= 0')
    safety = args.near_miss if args.near_miss is not None else 0.1 if args.safety else None
    if args.stall_window is not None and args.stall_window < 1:
        ap.error('--stall-window must be >= 1')
    progress = None
    if args.timeouts or args.stall_window is not None:
        progress = {} if args.stall_window is None else {'window': args.stall_window}
    if orca and (args.scan_noise is not None or args.beam_dropout is not None):
        ap.error('--scan-noise / --beam-dropout apply to --policy only: the ORCA baselines do not read the scan')
    noise_params = noise_from_arguments(ap, args)
    if orca and args.scan_delay is not None:
        ap.error('--scan-delay applies to --policy only: the ORCA baselines do not read the scan')
    latency_params = latency_from_arguments(ap, args)
    dynamics_params = dynamics_from_arguments(ap, args)
    localization_params = localization_from_arguments(ap, args)
    if localization_params is not None and (orca or args.hybrid):
        ap.error('--pose-error / --heading-error / --speed-error apply to --policy without --hybrid only: the ORCA '
                 'baselines and the hybrid driver read the true state')
    check_planner_arguments(ap, args, localization=localization_params is not None)
    steer = planner_from_arguments(args)
    hybrid_params = None
    if args.hybrid:
        hybrid_params = dict(HYBRID_DEFAULTS)
        for k, a in zip(('r_safe', 'r_risk', 'v_safe'), hybrid_args):
            if a is not None:
                hybrid_params[k] = a
        try:
            check_hybrid(COMMON['range_max'], v_max, **hybrid_params)
        except ValueError as e:
            ap.error(str(e))
    if args.scenario == 'circle':
        sc = make_scenario(args.scenario, robots_per_world=args.circle_robots, radius=args.circle_radius)
    elif args.scenario == 'random':
        sc = random_scenario_from_arguments(ap, args)
    elif args.scenario == 'arena':
        sc = arena_scenario_from_arguments(ap, args, pick=0)
    else:
        sc = make_scenario(args.scenario)
    if args.non_cooperative is not None and not 1 <= args.non_cooperative <= sc.robots_per_world:
        ap.error('--non-cooperative must be in 1..%d on %s' % (sc.robots_per_world, args.scenario))
    if args.crowd is not None and not 1 <= args.crowd <= sc.robots_per_world:
        ap.error('--crowd must be in 1..%d on %s' % (sc.robots_per_world, args.scenario))
    crowd_params = crowd_from_arguments(ap, args, v_max)
    dwa_params = dwa_from_arguments(ap, args)
    plan_tables = None
    if steer is not None:
        try:
            plan_tables = build_plan_tables(sc.map)
        except ValueError as e:
            ap.error('--%s: %s' % ('planner' if steer else 'geodesic', e))
    env = StageWorld(LASER_BEAM, index=0, scenario=sc, num_worlds=args.num_worlds, seed=args.seed,
                     auto_reset=AUTO_RESET[args.scenario])
    if dwa_params is not None:
        policy, controller = DwaController(env, dwa_params), 'dwa'
    elif args.baseline is not None:
        policy, controller = controller_from_arguments(env, args)
    else:
        policy = CNNPolicy(frames=LASER_HIST, action_space=2, max_batch=env.N)
        policy.load_state_dict(torch.load(args.policy, map_location='cuda'))
        controller = None
    if args.max_ticks is not None:
        max_ticks = args.max_ticks
    elif args.scenario == 'circle':
        max_ticks = CIRCLE_MAX_TICKS
    elif args.scenario in ('random', 'arena'):
        max_ticks = random_max_ticks(sc.layout.side)
    else:
        max_ticks = args.episodes * (sc.timeout + 1)
    nc = None
    if args.non_cooperative is not None:
        nc = NonCooperative(env, non_cooperative_mask(sc.robots_per_world, args.num_worlds, args.non_cooperative),
                            speed=args.non_cooperative_speed)
    crowd = None
    if crowd_params is not None:
        k, cp, crowd_map = crowd_params
        crowd = Crowd(env, non_cooperative_mask(sc.robots_per_world, args.num_worlds, k), cp, obstacles=crowd_map)
    masked = nc if nc is not None else crowd
    role, label = ('crowd', 'crowd  ') if crowd is not None else ('non_cooperative', 'non-cooperative  ')
    hy = Hybrid(env, **hybrid_params) if args.hybrid else None
    noise = Noise(env, noise_params) if noise_params is not None else None
    latency = Latency(env, latency_params) if latency_params is not None else None
    dynamics = Dynamics(env, dynamics_params) if dynamics_params is not None else None
    localization = Localization(env, localization_params) if localization_params is not None else None
    planner = Planner(env, steer, tables=plan_tables) if steer is not None else None
    out = evaluate(env, policy, args.episodes, max_ticks, check_every=args.check_every, non_cooperative=nc, hybrid=hy,
                   safety=safety, progress=progress, noise=noise, latency=latency, dynamics=dynamics,
                   localization=localization, crowd=crowd, planner=planner)

    def line(m, robots, role=''):
        f = lambda k: '%.3f +- %.3f' % m[k]
        print(('%s  ' % controller if controller else '') + role +
              '%s  robots %d  ticks %d  episodes %d  success %.4f  crash %.4f  time-out %.4f  unfinished %d  '
              'extra time %s s  extra distance %s m  average speed %s m/s'
              % (args.scenario, robots, out['ticks'], m['episodes'], m['success_rate'], m['crash_rate'],
                 m['timeout_rate'], m['unfinished'], f('extra_time'), f('extra_distance'), f('average_speed')))

    m = out['metrics']
    if noise is not None:
        ns = out['noise']
        print('noise  range sigma %g m  beam dropout %g  v gain sigma %g  w gain sigma %g  seed %d'
              % (ns['range_sigma'], ns['dropout'], ns['v_gain_sigma'], ns['w_gain_sigma'], ns['seed']))
    if latency is not None:
        ls = out['latency']
        print('latency  scan delay %d..%d ticks  command delay %d..%d ticks  (tick %g s)  seed %d'
              % (*ls['scan_delay'], *ls['command_delay'], env.cfg.dt, ls['seed']))
    if dynamics is not None:
        ds = out['dynamics']
        limit = lambda r, unit: 'off' if r[1] == 0 else ('%g' % r[0] if r[0] == r[1] else '%g..%g' % tuple(r)) + unit
        print('dynamics  linear accel limit %s  angular accel limit %s  (tick %g s)  seed %d'
              % (limit(ds['linear'], ' m/s^2'), limit(ds['angular'], ' rad/s^2'), env.cfg.dt, ds['seed']))
    if localization is not None:
        lo = out['localization']
        sig = lambda r, unit: 'off' if r[1] == 0 else ('%g' % r[0] if r[0] == r[1] else '%g..%g' % tuple(r)) + unit
        print('localization  pose sigma %s  heading sigma %s  correlation time %g s  speed sigma %g m/s %g rad/s  '
              'seed %d' % (sig(lo['pose_sigma'], ' m'), sig(lo['heading_sigma'], ' rad'), lo['correlation_time'],
                           *lo['speed_sigma'], lo['seed']))
    line(m, env.N)
    if dwa_params is not None:
        print('dwa  fallback share %.4f of robot-ticks (no admissible candidate: (0, 0) commanded)'
              % out['dwa']['fallback_share'])
    if masked is not None:
        k = int(masked.mask.count_nonzero())
        line(out['by_role']['cooperative'], env.N - k, 'cooperative  ')
        line(out['by_role'][role], k, label)
    if planner is not None and planner.steer:
        p = out['planner']
        print('planner over %d %srobot-ticks: goal visible %.4f  waypoint %.4f  no plan %.4f  (%d components, '
              'largest field %d cells)' % (p['robot_ticks'], 'cooperative ' if masked is not None else '',
                                           p['goal_visible'], p['waypoint'], p['no_plan'], p['components'],
                                           p['max_area']))

    def geodesic_line(g, role=''):
        print('geodesic  %sreached with a path %d  mean geodesic length %.3f m  extra geodesic distance %.3f +- %.3f m  '
              'no path %d' % (role, g['reached'], g['mean_length'], *g['extra_geodesic_distance'], g['no_path']))

    if planner is not None:
        geodesic_line(out['geodesic'])
        if masked is not None:
            geodesic_line(out['geodesic_by_role']['cooperative'], 'cooperative  ')
            geodesic_line(out['geodesic_by_role'][role], label)
    if hy is not None:
        s = out['modes']
        print('hybrid modes over %d %srobot-ticks: policy %.4f  driver %.4f  safe %.4f'
              % (s['agent_ticks'], 'cooperative ' if masked is not None else '', s['policy'], s['driver'], s['safe']))

    def safety_line(m, role=''):
        f = lambda k: '%.3f +- %.3f' % m[k]
        print('safety  %scrashes static %d  robot %d (both in range %d%s)  robot share %.4f  min separation %s m  '
              'min clearance %s m  near-miss rate %.4f (< %g m)  least separation %.3f m'
              % (role, m['crash_static'], m['crash_robot'], m['crash_both_in_range'],
                 ', into %s %d' % (label.strip(), m['crash_into_masked']) if masked is not None else '',
                 m['crash_robot_share'], f('min_separation_reached'), f('min_clearance_reached'), m['near_miss_rate'],
                 safety, m['min_separation']))

    if safety is not None:
        safety_line(out['safety'])
        if masked is not None:
            safety_line(out['safety_by_role']['cooperative'], 'cooperative  ')
            safety_line(out['safety_by_role'][role], label)

    def progress_line(m, role=''):
        f = lambda k: '%.3f +- %.3f' % m[k]
        group = lambda g, name, n: ('%s %d: frozen %d  stalled %d  slow %d  robot near %d  closest %s m'
                                    % (name, n, m[g + '_frozen'], m[g + '_stalled'], m[g + '_slow'],
                                       m[g + '_robot_near'], f(g + '_closest')))
        print('progress  %s%s  |  %s  |  still share %.4f  rotation per reached %s rad  (window %d ticks)'
              % (role, group('timeout', 'time-outs', m['timeouts']), group('unfinished', 'unfinished', m['unfinished']),
                 m['still_share'], f('rotation_reached'), out['progress_tracker'].params['window']))

    if progress is not None:
        progress_line(out['progress'])
        if masked is not None:
            progress_line(out['progress_by_role']['cooperative'], 'cooperative  ')
            progress_line(out['progress_by_role'][role], label)
    arenas = None
    if args.per_arena:
        arenas = per_arena(out['partials'], sc.layout, int(env.cfg.world_offset))
        seen = [r for r in arenas if r['metrics']['episodes']]
        low = sorted(seen, key=lambda r: (r['metrics']['success_rate'], r['arena']))[:10]
        print('per arena (world w in arena w mod %d), lowest success of %d arenas with episodes:'
              % (sc.layout.count, len(seen)))
        for r in low:
            ma = r['metrics']
            print('  arena %3d  cells %5d  worlds %d  episodes %d  success %.4f  crash %.4f  time-out %.4f  '
                  'unfinished %d' % (r['arena'], r['cells'], r['worlds'], ma['episodes'], ma['success_rate'],
                                     ma['crash_rate'], ma['timeout_rate'], ma['unfinished']))
    if args.json:
        perturbations = (('noise', NOISE_FLAGS), ('latency', LATENCY_FLAGS), ('dynamics', DYNAMICS_FLAGS),
                         ('localization', LOCALIZATION_FLAGS))
        hidden = (() if safety is not None else ('safety', 'near_miss')) + \
            (() if progress is not None else ('timeouts', 'stall_window')) + \
            tuple(f[2:].replace('-', '_') for name, flags in perturbations if name not in out for f in flags) + \
            (() if crowd is not None else ('crowd',) + tuple(f[2:].replace('-', '_') for f in CROWD_FLAGS)) + \
            (() if dwa_params is not None else tuple(f[2:].replace('-', '_') for f in DWA_FLAGS)) + \
            (() if planner is not None else ('planner', 'geodesic'))
        shown = {k: v for k, v in vars(args).items() if k not in hidden}
        res = {'args': shown, 'controller': controller or 'policy', 'robots': env.N,
               'ticks': out['ticks'], 'metrics': m,
               'columns': list(COLUMNS), 'totals': out['totals'].tolist(),
               'partials': out['partials'].tolist()}
        res.update((name, out[name]) for name, _ in perturbations if name in out)
        if crowd is not None:
            res['crowd'] = crowd.settings()
        if dwa_params is not None:
            res['dwa'] = out['dwa']
        if planner is not None:
            if planner.steer:
                res['planner'] = out['planner']
            res['geodesic'] = {'metrics': out['geodesic'], 'columns': list(GEODESIC_COLUMNS),
                               'totals': out['geodesic_totals'].tolist(), 'partials': out['geodesic_partials'].tolist()}
            if masked is not None:
                res['geodesic']['by_role'] = out['geodesic_by_role']
                res['geodesic']['partials_split'] = out['geodesic_partials_split'].tolist()
        if masked is not None:
            res['by_role'] = out['by_role']
            res['partials_split'] = out['partials_split'].tolist()
        if arenas is not None:
            res['per_arena'] = [{'arena': r['arena'], 'cells': r['cells'], 'worlds': r['worlds'],
                                 **{k: r['metrics'][k] for k in ('episodes', 'success_rate', 'crash_rate',
                                                                 'timeout_rate', 'unfinished')}} for r in arenas]
        if hy is not None:
            res['modes'] = out['modes']
            res['mode_counts'] = out['mode_counts'].tolist()
        if safety is not None:
            res['safety'] = {'near_miss': safety, 'metrics': out['safety'], 'columns': list(SAFETY_COLUMNS),
                             'totals': out['safety_totals'].tolist(), 'partials': out['safety_partials'].tolist()}
            if masked is not None:
                res['safety']['by_role'] = out['safety_by_role']
                res['safety']['partials_split'] = out['safety_partials_split'].tolist()
        if progress is not None:
            res['progress'] = {'params': out['progress_tracker'].params, 'metrics': out['progress'],
                               'columns': list(PROGRESS_COLUMNS), 'totals': out['progress_totals'].tolist(),
                               'partials': out['progress_partials'].tolist()}
            if masked is not None:
                res['progress']['by_role'] = out['progress_by_role']
                res['progress']['partials_split'] = out['progress_partials_split'].tolist()
        with open(args.json, 'w') as fh:
            json.dump(res, fh, indent=1)
    return out


if __name__ == '__main__':
    main()
