#!/usr/bin/env python
"""Stage-1 trainer on the H100-native stack (drop-in for the reference's ppo_stage1.py).

Same hyper-parameters, log files and checkpoint names; `mpiexec -np 24` is replaced by one process per GPU:
    python ppo_stage1.py --num-worlds 43                       # 1 GPU, 43 x 24 = 1032 robots
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 ppo_stage1.py --num-worlds 43
"""
import argparse
import logging
import os
import socket
import sys

import torch

from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
from rl_collision_avoidance_b200.model.ppo import setup_ppo_log
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


def main(stage=1, world_cls=StageWorld, num_env=NUM_ENV, batch_size=BATCH_SIZE, epoch=EPOCH, ckpt='stage1_2.pth'):
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-worlds', type=int, default=1, help='independent worlds per GPU (x %d robots each)' % num_env)
    ap.add_argument('--updates', type=int, default=None, help='stop after this many PPO updates')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--policy-path', default='policy')
    ap.add_argument('--resume', default=None, help='checkpoint written by this trainer (e.g. policy/Stage1_40): restores the\n'
                    'weights and, from <file>.trainer, the Adam moments / step and the sampling counter')
    ap.add_argument('--scenario', default=None, choices=[None, 'stage1', 'stage2', 'circle'],
                    help='override the world (e.g. circle: BASELINE config 4 trains on circle.world)')
    args = ap.parse_args()
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
    device = 'cuda:%d' % local_rank
    if args.scenario == 'circle':
        from rl_collision_avoidance_b200.circle_world import StageWorld as world_cls   # noqa: N813
        num_env = 50
    env = world_cls(LASER_BEAM, index=0, num_env=num_env, num_worlds=args.num_worlds, device=device, seed=args.seed,
                    auto_reset=1 if stage == 1 else 2, world_offset=rank * args.num_worlds)
    action_bound = [[0, -1], [1, 1]]
    policy = CNNPolicy(frames=LASER_HIST, action_space=2, device=device, seed=args.seed, max_batch=max(batch_size, env.N))
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
    if args.resume:
        policy.load_state_dict(torch.load(args.resume, map_location=device))
        extra = args.resume + '.trainer'
        if os.path.exists(extra):
            st = torch.load(extra, map_location=device)
            opt.load_state_dict(st['optimizer'])
            policy.sample_counter = int(st.get('sample_counter', 0))
            start_update = int(st.get('update', 0))              # checkpoint names continue instead of overwriting
            if logger:
                logger.info('resumed from %s (update %d, Adam step %d)' % (args.resume, st.get('update', -1), opt.step_count))
    hp = dict(HORIZON=HORIZON, GAMMA=GAMMA, LAMDA=LAMDA, BATCH_SIZE=batch_size, EPOCH=epoch, COEFF_ENTROPY=COEFF_ENTROPY,
              CLIP_VALUE=CLIP_VALUE, NUM_ENV=num_env, OBS_SIZE=OBS_SIZE, ACT_SIZE=ACT_SIZE, LASER_HIST=LASER_HIST,
              MAX_EPISODES=MAX_EPISODES)
    try:
        stats = run(env=env, policy=policy, policy_path=args.policy_path, action_bound=action_bound, optimizer=opt, hp=hp,
                    logger=logger, logger_cal=logger_cal, stage=stage, max_updates=args.updates, process_group=pg, rank=rank,
                    start_update=start_update)
        if rank == 0 and stats:
            s = stats[-1]
            print('update %d: rollout %.3fs update %.3fs -> %.0f agent-steps/s per GPU; mean ep reward %.2f' %
                  (s['update'], s['rollout_s'], s['update_s'], s['agent_steps_per_s'], s['mean_ep_reward']))
    except KeyboardInterrupt:
        pass
    finally:
        if world_size > 1:
            import torch.distributed as dist
            dist.destroy_process_group()


if __name__ == '__main__':
    main()
