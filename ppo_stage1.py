#!/usr/bin/env python
"""Stage-1 trainer on the H100-native stack (drop-in for the reference's ppo_stage1.py).

Same hyper-parameters, log files and checkpoint names; `mpiexec -np 24` is replaced by one process per GPU:
    python ppo_stage1.py --num-worlds 43                       # 1 GPU, 43 x 24 = 1032 robots
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 ppo_stage1.py --num-worlds 43
Fine-tuning on random layouts (DESIGN.md §9k) runs through ppo_stage2.py --scenario random, on generated obstacle
arenas (DESIGN.md §9v) through ppo_stage2.py --scenario arena, and on a mix of scenarios (DESIGN.md §9l) through
ppo_stage2.py --mix.  --scan-noise SIGMA_M, --beam-dropout P and --action-noise SIGMA_V[,SIGMA_W]
train under lidar and actuation noise (DESIGN.md §9p), with any scenario or mix.  --scan-delay T[,T_MAX] and
--command-delay T[,T_MAX] train under sensing and command latency, in ticks of 0.1 s (DESIGN.md §9q).
--accel-limit A[,A_MAX] and --angular-accel-limit B[,B_MAX] train under acceleration limits, in m/s^2 and rad/s^2
(DESIGN.md §9r).  --pose-error S[,S_MAX], --heading-error S[,S_MAX], --pose-error-time T and --speed-error SV[,SW]
train under localization error in the policy's local goal and speed (DESIGN.md §9s).  --non-cooperative K
[--non-cooperative-speed S] puts K straight-to-goal drivers into every world (DESIGN.md §9h), --crowd K (with
--crowd-speed, --crowd-ignores-robots, --crowd-map, --crowd-strength, --crowd-range, --crowd-side-bias) K social-force
crowd agents (DESIGN.md §9t); either way their rows are left out of every PPO update, with any scenario or mix.
--planner trains with the global planner (DESIGN.md §9x): the policy reads a line-of-sight waypoint on the geodesic path
as its local goal and the reward pays geodesic progress; --planner-reward straight keeps the tick's straight-line
reward.  Stage 1, stage 2 and the arenas, alone or mixed; not with localization error, random layouts or the circle.
--arena-curriculum [--curriculum-decay L] [--curriculum-uniform E] draws the arena of each re-layout by an automatic
curriculum (DESIGN.md §9z): per-arena success tallied on the device, arenas the policy neither always nor never solves
drawn more often.  --scenario arena or an arena component of --mix.
"""
import argparse
import logging
import os
import socket
import sys

import torch

from rl_collision_avoidance_b200.crowd import add_crowd_arguments, crowd_from_arguments, \
    non_cooperative_from_arguments
from rl_collision_avoidance_b200.curriculum import CurriculumParams, check_params
from rl_collision_avoidance_b200.dynamics import add_dynamics_arguments, dynamics_from_arguments
from rl_collision_avoidance_b200.latency import add_latency_arguments, latency_from_arguments
from rl_collision_avoidance_b200.localization import add_localization_arguments, localization_from_arguments
from rl_collision_avoidance_b200.mix import MIX_AUTO_RESET, parse_mix, plan
from rl_collision_avoidance_b200.model.diagnostics import check_target_kl, setup_diag_log
from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
from rl_collision_avoidance_b200.model.ppo import setup_ppo_log
from rl_collision_avoidance_b200.noise import add_noise_arguments, noise_from_arguments
from rl_collision_avoidance_b200.planner import build_plan_tables
from rl_collision_avoidance_b200.scenarios import COMMON, add_arena_arguments, add_random_arguments, \
    arena_scenario_from_arguments, check_arena_arguments, check_random_arguments, make_scenario, \
    random_scenario_from_arguments
from rl_collision_avoidance_b200.stage_world import StageWorld as RandomWorld
from rl_collision_avoidance_b200.stage_world1 import StageWorld
from rl_collision_avoidance_b200.trainer import run

MAX_EPISODES = 5000
LASER_BEAM = 512
LASER_HIST = 3
HORIZON = 128
GAMMA = 0.99
LAMDA = 0.95
BATCH_SIZE = 1024
EPOCH = 2
COEFF_ENTROPY = 5e-4
CLIP_VALUE = 0.1
NUM_ENV = 24
OBS_SIZE = 512
ACT_SIZE = 2
LEARNING_RATE = 5e-5


def make_loggers():
    hostname = socket.gethostname()
    d = './log/' + hostname
    os.makedirs(d, exist_ok=True)
    logger = logging.getLogger('mylogger')
    logger.setLevel(logging.INFO)
    fh = logging.FileHandler(d + '/output.log', mode='a')
    fh.setFormatter(logging.Formatter('%(asctime)s - %(levelname)s - %(message)s'))
    logger.addHandler(fh)
    logger.addHandler(logging.StreamHandler(sys.stdout))
    logger_cal = logging.getLogger('loggercal')
    logger_cal.setLevel(logging.INFO)
    logger_cal.addHandler(logging.FileHandler(d + '/cal.log', mode='a'))
    setup_ppo_log()
    return logger, logger_cal


def mix_components(mix, sc, rank, arena_sc=None):
    """The Components of a parsed --mix on GPU `rank`: stage 2's 44 robots per world, the shipped circle's 50, the
    random scenario `sc`'s K (sc is None without a random component) and the arena scenario `arena_sc`'s K."""
    robots = {'stage2': 44, 'circle': 50, 'random': sc.robots_per_world if sc is not None else None,
              'arena': arena_sc.robots_per_world if arena_sc is not None else None}
    return plan(mix, robots, rank)


def make_component_env(c, sc, device, seed, arena_sc=None):
    """The env handle of mix component `c`, built as a single-scenario run of that scenario builds it."""
    kw = dict(num_worlds=c.worlds, device=device, seed=seed, auto_reset=MIX_AUTO_RESET[c.name],
              world_offset=c.world_offset)
    if c.name == 'stage2':
        from rl_collision_avoidance_b200.stage_world2 import StageWorld as Stage2World
        return Stage2World(LASER_BEAM, index=0, num_env=c.robots_per_world, **kw)
    if c.name == 'circle':
        from rl_collision_avoidance_b200.circle_world import StageWorld as CircleWorld
        return CircleWorld(LASER_BEAM, index=0, num_env=c.robots_per_world, **kw)
    if c.name == 'arena':
        return RandomWorld(LASER_BEAM, index=0, scenario=arena_sc, **kw)
    return RandomWorld(LASER_BEAM, index=0, scenario=sc, **kw)


def component_summary(c, stats):
    """One line per mix component over every update of the run: episodes, successes, crashes, mean episode reward."""
    rows = [s['by_scenario'][c.name] for s in stats]
    n = sum(r['episodes'] for r in rows)
    count = lambda key: sum(round(r[key] * r['episodes']) for r in rows if r['episodes'])
    reward = sum(r['mean_ep_reward'] * r['episodes'] for r in rows if r['episodes'])
    return ('  %s: %d worlds x %d robots, columns [%d, %d): %d episodes, %d reached the goal, %d crashed, '
            'mean ep reward %.2f' % (c.name, c.worlds, c.robots_per_world, c.cols[0], c.cols[1], n,
                                     count('success_rate'), count('crash_rate'), reward / n if n else float('nan')))


def main(stage=1, world_cls=StageWorld, num_env=NUM_ENV, batch_size=BATCH_SIZE, epoch=EPOCH, ckpt='stage1_2.pth',
         argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-worlds', type=int, default=None,
                    help='independent worlds per GPU (x %d robots each; default 1)' % num_env)
    ap.add_argument('--updates', type=int, default=None, help='stop after this many PPO updates')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--policy-path', default='policy')
    ap.add_argument('--resume', default=None, help='checkpoint written by this trainer (e.g. policy/Stage1_40): restores the\n'
                    'weights and, from <file>.trainer, the Adam moments / step and the sampling counter')
    ap.add_argument('--scenario', default=None, choices=[None, 'stage1', 'stage2', 'circle', 'random', 'arena'],
                    help='override the world (e.g. circle: BASELINE config 4 trains on circle.world; random: a new '
                         'layout in a world whenever all its robots have ended their episodes, stage 2 only; arena: '
                         'the same in a newly drawn generated obstacle arena)')
    ap.add_argument('--mix', default=None, metavar='NAME:W,...',
                    help='train on several scenarios in one run (stage 2 only; DESIGN.md §9l): world counts per GPU of '
                         'stage2, circle, random and arena, e.g. stage2:31,random:128,circle:14')
    ap.add_argument('--diagnostics', action='store_true',
                    help='write the health of every PPO update to log/<host>/diag.log (DESIGN.md §9n): approximate KL, '
                         'clip fraction, explained variance, ratio extremes, action saturation, gradient norms')
    ap.add_argument('--target-kl', type=float, default=None, metavar='X',
                    help='skip the remaining epochs of an update once an epoch moved the policy by more than X '
                         '(approx_kl_k3; finite and > 0; implies --diagnostics)')
    add_random_arguments(ap, timeout=True)
    add_arena_arguments(ap, timeout=True)
    add_noise_arguments(ap)
    add_latency_arguments(ap)
    add_dynamics_arguments(ap)
    add_localization_arguments(ap)
    add_crowd_arguments(ap, non_cooperative=True)
    ap.add_argument('--planner', action='store_true',
                    help='train with the global planner (DESIGN.md §9x): a waypoint on the geodesic path as the '
                         "policy's local goal where the goal is out of sight, and a geodesic progress reward")
    ap.add_argument('--planner-reward', default=None, choices=('geodesic', 'straight'),
                    help='with --planner: geodesic (default) shapes the reward by geodesic progress, straight keeps '
                         "the tick's straight-line reward")
    ap.add_argument('--arena-curriculum', action='store_true',
                    help='draw the arena of every re-layout by an automatic curriculum (DESIGN.md §9z): arenas whose '
                         'recent success rate is neither near 0 nor near 1 more often')
    ap.add_argument('--curriculum-decay', type=float, default=None, metavar='L',
                    help='with --arena-curriculum: weight of the per-arena counts before each update, in [0, 1) '
                         '(default %g)' % CurriculumParams.decay)
    ap.add_argument('--curriculum-uniform', type=float, default=None, metavar='E',
                    help='with --arena-curriculum: share of every arena\'s score independent of its outcomes, in [0, 1] '
                         '(default %g)' % CurriculumParams.uniform)
    args = ap.parse_args(argv)
    noise = noise_from_arguments(ap, args)
    latency = latency_from_arguments(ap, args)
    dynamics = dynamics_from_arguments(ap, args)
    localization = localization_from_arguments(ap, args)
    non_cooperative = non_cooperative_from_arguments(ap, args, COMMON['v_max'])
    crowd = crowd_from_arguments(ap, args, COMMON['v_max'])
    if args.target_kl is not None:
        try:
            args.target_kl = check_target_kl(args.target_kl)
        except ValueError as e:
            ap.error('--target-kl: %s' % e)
        args.diagnostics = True
    mix = None
    if args.mix is not None:
        if stage != 2:
            ap.error('--mix trains with ppo_stage2.py: every component trains with stage 2\'s update')
        if args.scenario is not None or args.num_worlds is not None:
            ap.error('--mix gives the scenarios and their world counts: drop --scenario and --num-worlds')
        try:
            mix = parse_mix(args.mix)
        except ValueError as e:
            ap.error(str(e))
    if args.num_worlds is None:
        args.num_worlds = 1
    random_in_mix = mix is not None and any(name == 'random' for name, _ in mix)
    arena_in_mix = mix is not None and any(name == 'arena' for name, _ in mix)
    check_arena_arguments(ap, args, arena_component=arena_in_mix)
    check_random_arguments(ap, args, random_component=random_in_mix)
    sc = arena_sc = None
    if args.scenario == 'random' or random_in_mix:
        if stage != 2:
            ap.error('--scenario random trains with ppo_stage2.py: its layouts are per world, and stage 1 re-spawns '
                     'each robot on its own')
        sc = random_scenario_from_arguments(ap, args)
    if args.scenario == 'arena' or arena_in_mix:
        if stage != 2:
            ap.error('--scenario arena trains with ppo_stage2.py: its layouts are per world, and stage 1 re-spawns '
                     'each robot on its own')
        arena_sc = arena_scenario_from_arguments(ap, args, pick=1)
        if mix is None:
            sc = arena_sc
    curriculum = None
    if args.arena_curriculum:
        if args.scenario != 'arena' and not arena_in_mix:
            ap.error('--arena-curriculum needs --scenario arena or an arena component of --mix')
        try:
            curriculum = check_params(CurriculumParams(
                CurriculumParams.decay if args.curriculum_decay is None else args.curriculum_decay,
                CurriculumParams.uniform if args.curriculum_uniform is None else args.curriculum_uniform))
        except ValueError as e:
            ap.error('--arena-curriculum: %s' % e)
    elif args.curriculum_decay is not None or args.curriculum_uniform is not None:
        ap.error('--curriculum-decay / --curriculum-uniform apply with --arena-curriculum only')
    planner = planner_tables = None
    if args.planner_reward is not None and not args.planner:
        ap.error('--planner-reward needs --planner')
    if args.planner:
        if localization is not None:
            ap.error('--planner plans from the true pose; localization error needs a planner on the believed pose')
        names = [name for name, _ in mix] if mix is not None else \
            [args.scenario or ('stage1' if stage == 1 else 'stage2')]
        planner_tables = []                      # one per env, in the order the envs are built below
        for name in names:
            m = sc.map if name == 'random' else arena_sc.map if name == 'arena' else make_scenario(name).map
            try:
                planner_tables.append(build_plan_tables(m))
            except ValueError as e:
                ap.error('--planner on %s: %s' % (name, e))
        planner = args.planner_reward or 'geodesic'
    rank = int(os.environ.get('RANK', '0'))
    world_size = int(os.environ.get('WORLD_SIZE', '1'))
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local_rank)
    pg = None
    if world_size > 1:
        import torch.distributed as dist
        dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
        pg = True
    logger, logger_cal = make_loggers() if rank == 0 else (None, None)
    if rank == 0 and args.diagnostics:
        setup_diag_log()
    device = 'cuda:%d' % local_rank
    if args.scenario == 'circle':
        from rl_collision_avoidance_b200.circle_world import StageWorld as world_cls   # noqa: N813
        num_env = 50
    comps = None
    if mix is not None:
        comps = mix_components(mix, sc, rank, arena_sc)
        env = [make_component_env(c, sc, device, args.seed, arena_sc) for c in comps]
    elif sc is not None:
        env = RandomWorld(LASER_BEAM, index=0, scenario=sc, num_worlds=args.num_worlds, device=device, seed=args.seed,
                          auto_reset=0, world_offset=rank * args.num_worlds)
        num_env = sc.robots_per_world
    else:
        env = world_cls(LASER_BEAM, index=0, num_env=num_env, num_worlds=args.num_worlds, device=device,
                        seed=args.seed, auto_reset=1 if stage == 1 else 2, world_offset=rank * args.num_worlds)
    masked_k = non_cooperative[0] if non_cooperative is not None else crowd[0] if crowd is not None else None
    least_r = min(e.cfg.robots_per_world for e in (env if comps is not None else [env]))
    if masked_k is not None and masked_k > least_r:
        ap.error('--%s must be in 1..%d: a world has %d robots'
                 % ('crowd' if crowd is not None else 'non-cooperative', least_r, least_r))
    action_bound = [[0, -1], [1, 1]]
    n_agents = sum(e.N for e in env) if comps is not None else env.N
    policy = CNNPolicy(frames=LASER_HIST, action_space=2, device=device, seed=args.seed, max_batch=max(batch_size, n_agents))
    policy.sample_seed = args.seed * 1000003 + rank              # every rank draws its own action noise
    opt = Adam(policy.parameters(), lr=LEARNING_RATE)
    if world_size > 1 and os.environ.get('RLCA_DP_PEER', '1') == '1':
        # gradient sum + Adam + broadcast as one kernel over NVLink peer memory; NCCL all-reduce + Adam otherwise
        try:
            from rl_collision_avoidance_b200.parallel import PeerAdam
            peer = PeerAdam.attach(policy, opt)
            if logger:
                logger.info('data-parallel optimizer step over peer memory (%s)' % ('NVLS multicast' if peer.nvls else 'P2P'))
        except Exception as e:                      # no symmetric memory on this box: the NCCL path is always there
            if logger:
                logger.info('peer-memory optimizer step unavailable (%r): NCCL all-reduce + Adam' % (e,))
    os.makedirs(args.policy_path, exist_ok=True)
    file = args.policy_path + '/' + ckpt
    if os.path.exists(file):
        if logger:
            logger.info('####################################')
            logger.info('############Loading Model###########')
            logger.info('####################################')
        policy.load_state_dict(torch.load(file, map_location=device))
    elif logger:
        logger.info('#####################################')
        logger.info('############Start Training###########')
        logger.info('#####################################')
    start_update = 0
    curriculum_state = None
    if args.resume:
        policy.load_state_dict(torch.load(args.resume, map_location=device))
        extra = args.resume + '.trainer'
        if os.path.exists(extra):
            st = torch.load(extra, map_location=device)
            opt.load_state_dict(st['optimizer'])
            policy.sample_counter = int(st.get('sample_counter', 0))
            start_update = int(st.get('update', 0))              # checkpoint names continue instead of overwriting
            if curriculum is not None:
                curriculum_state = st.get('curriculum')
            if logger:
                logger.info('resumed from %s (update %d, Adam step %d)' % (args.resume, st.get('update', -1), opt.step_count))
    hp = dict(HORIZON=HORIZON, GAMMA=GAMMA, LAMDA=LAMDA, BATCH_SIZE=batch_size, EPOCH=epoch, COEFF_ENTROPY=COEFF_ENTROPY,
              CLIP_VALUE=CLIP_VALUE, NUM_ENV=num_env, OBS_SIZE=OBS_SIZE, ACT_SIZE=ACT_SIZE, LASER_HIST=LASER_HIST,
              MAX_EPISODES=MAX_EPISODES)
    try:
        stats = run(env=env, policy=policy, policy_path=args.policy_path, action_bound=action_bound, optimizer=opt, hp=hp,
                    logger=logger, logger_cal=logger_cal, stage=stage, max_updates=args.updates, process_group=pg, rank=rank,
                    start_update=start_update, diagnostics=args.diagnostics, target_kl=args.target_kl, noise=noise,
                    latency=latency, dynamics=dynamics, localization=localization, non_cooperative=non_cooperative,
                    crowd=crowd, planner=planner, planner_tables=planner_tables, curriculum=curriculum,
                    curriculum_state=curriculum_state)
        if rank == 0 and stats:
            s = stats[-1]
            print('update %d: rollout %.3fs update %.3fs -> %.0f agent-steps/s per GPU; mean ep reward %.2f' %
                  (s['update'], s['rollout_s'], s['update_s'], s['agent_steps_per_s'], s['mean_ep_reward']))
            for c in comps or ():
                print(component_summary(c, stats))
            if 'planner' in s:
                print('last update, planner: %s' % ', '.join('%s %.3f' % (k, v) for k, v in s['planner'].items()
                                                             if k != 'robot_ticks'))
            if 'curriculum' in s:
                cu = s['curriculum']
                print('last update, curriculum: %d arenas, effective %.1f, draw share max %.4f min %.4f, %d episodes '
                      'folded in' % (cu['arenas'], cu['effective_arenas'], cu['max_share'], cu['min_share'],
                                     cu['episodes']))
            if 'by_role' in s:
                for role, r in s['by_role'].items():
                    print('last update, %s: %d episodes, success %.3f, crash %.3f'
                          % (role, r['episodes'], r['success_rate'], r['crash_rate']))
    except KeyboardInterrupt:
        pass
    finally:
        if world_size > 1:
            import torch.distributed as dist
            dist.destroy_process_group()


if __name__ == '__main__':
    main()
