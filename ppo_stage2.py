#!/usr/bin/env python
"""Stage-2 trainer (drop-in for /root/reference/ppo_stage2.py): testenv map + polygon obstacles, 44 robots per
world, group-synchronous episodes, filtered idle transitions, BATCH_SIZE 512, EPOCH 4, drop_last.
Curriculum: copy a stage-1 checkpoint to policy/stage2.pth (README.md:18 of the reference).

--scenario random fine-tunes on random layouts (DESIGN.md §9k): --random-robots K robots per world in a --random-side
S m square on circle.world's map, a new layout in a world whenever all its robots have ended their episodes, episodes
timing out after --random-timeout ticks (default 3 ceil(S sqrt(2) / (v_max dt)), 426 for the default 10 m square):
    mkdir -p policy && cp tests/golden/checkpoints/stage2.pth policy/stage2.pth
    python ppo_stage2.py --scenario random --random-robots 16 --num-worlds 256 --updates 100

--scenario arena fine-tunes among static obstacles (DESIGN.md §9v): --arena-robots K robots per world in one of
--arena-count generated walled arenas with --arena-obstacles LO,HI random obstacles each, an arena drawn anew at every
re-layout; --arena-seed picks the arenas, so evaluating with another seed tests on held-out arenas:
    python ppo_stage2.py --scenario arena --arena-robots 8 --num-worlds 256 --updates 100 --arena-seed 0

--mix trains on several scenarios in one run (DESIGN.md §9l): stage 2, the circle and random layouts side by side,
world counts per GPU, every PPO update over all of them (the --random-* flags shape the random component, the --arena-*
flags the arena component):
    python ppo_stage2.py --mix stage2:31,random:128,circle:14 --random-robots 16 --updates 100
    python ppo_stage2.py --mix stage2:31,arena:128 --updates 100

--crowd K puts K social-force crowd agents into every world (DESIGN.md §9t), --non-cooperative K K straight-to-goal
drivers (§9h); their rows are left out of every PPO update:
    python ppo_stage2.py --scenario random --random-robots 16 --num-worlds 128 --updates 100 --crowd 4 --crowd-map
"""
from ppo_stage1 import main
from rl_collision_avoidance_b200.stage_world2 import StageWorld

NUM_ENV = 44
BATCH_SIZE = 512
EPOCH = 4

if __name__ == '__main__':
    main(stage=2, world_cls=StageWorld, num_env=NUM_ENV, batch_size=BATCH_SIZE, epoch=EPOCH, ckpt='stage2.pth')
