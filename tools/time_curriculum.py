#!/usr/bin/env python
"""The cost numbers of DESIGN.md §9z, with CUDA events round every call, in two alternating passes:
  - the re-layout launch after a tick: rlca_layout_arena_weighted_respawn (tally + weighted re-layout, unequal weights)
    against rlca_layout_arena_respawn with pick 1, at 256 x 8 and 1024 x 16 on 64 arenas of 10 m, once with every
    world re-laid (every robot latched, every row an ended episode) and once with none (no robot latched);
  - rlca_arena_curriculum_update at T = 64 and 576;
  - trainer.run on arenas (256 worlds x 8 robots, pick 1, from stage2.pth): agent-steps/s without and with
    --arena-curriculum, the mean of updates 2 and 3 of a 3-update run.
Prints the card, power limit and maximum SM clock first.

    python tools/time_curriculum.py
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200 import _lib  # noqa: E402
from rl_collision_avoidance_b200.curriculum import ArenaCurriculum, CurriculumParams  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402

CALLS = 200
STAGE2 = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')


def _per_call_us(fn, before=None, calls=CALLS):
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(calls)]
    for _ in range(10):
        if before:
            before()
        fn()
    for e0, e1 in evs:
        if before:
            before()
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return 1e3 * float(np.mean([e0.elapsed_time(e1) for e0, e1 in evs]))


def relayout_times(K, W):
    """{(launch, case): us} of the two re-layout launches at W worlds x K robots."""
    sc = make_scenario('arena', robots_per_world=K, arenas=64, pick=1)
    env = StageWorld(512, scenario=sc, num_worlds=W, seed=0, auto_reset=0)
    env.reset_world()
    env.random_layout()
    cur = ArenaCurriculum(env, CurriculumParams())
    g = torch.Generator(device='cuda').manual_seed(0)
    cur.cdf[1:] = torch.cumsum(torch.randint(1, 1 << 20, (64,), device='cuda', generator=g), 0)
    env.curriculum = None
    meta = env.state['meta']
    saved = {k: v.clone() for k, v in env.state.items()}
    flags = torch.zeros(env.N, 4, dtype=torch.uint8, device='cuda')
    st = env._state_struct(env._cur)
    p = lambda t: C.c_void_p(t.data_ptr())
    stream = env._stream()
    plain = lambda: _lib.check(env.lib.rlca_layout_arena_respawn(
        C.byref(env.cfg), C.byref(env._layout_params), C.byref(env._arena), 1, C.byref(st), p(flags), p(env.live),
        p(env._relayout_status), stream))
    weighted = lambda: _lib.check(env.lib.rlca_layout_arena_weighted_respawn(
        C.byref(env.cfg), C.byref(env._layout_params), C.byref(env._arena), C.byref(cur.struct), None, C.byref(st),
        p(flags), p(env.live), p(env._relayout_status), stream))
    out = {}
    for case, latched in (('every world re-laid', 1), ('none re-laid', 0)):
        def before(latched=latched):
            for k, v in saved.items():
                env.state[k].copy_(v)
            meta[:, 3] = latched
            flags.zero_()
            flags[:, 0] = latched
            flags[:, 2] = latched
        for _ in range(2):
            for name, fn in (('rlca_layout_arena_respawn pick 1', plain),
                             ('rlca_layout_arena_weighted_respawn', weighted)):
                out.setdefault((name, case), []).append(_per_call_us(fn, before))
    return {k: min(v) for k, v in out.items()}


def update_times():
    out = {}
    for T in (64, 576):
        bufs = dict(cdf=torch.zeros(T + 1, dtype=torch.int64, device='cuda'),
                    world_arena=torch.zeros(1, dtype=torch.int32, device='cuda'),
                    pending=torch.randint(0, 50, (2 * T,), dtype=torch.int32, device='cuda'),
                    E=torch.rand(T, device='cuda') * 100, S=torch.rand(T, device='cuda') * 50)
        st = _lib.ArenaCurriculum(T, *(C.c_void_p(bufs[k].data_ptr()) for k in ('cdf', 'world_arena', 'pending',
                                                                                 'E', 'S')))
        lib = _lib.load()
        fn = lambda: _lib.check(lib.rlca_arena_curriculum_update(C.byref(st), 0.9, 0.1, None))
        out[T] = min(_per_call_us(fn) for _ in range(2))
    return out


def train_rate(curriculum):
    """Mean agent-steps/s of updates 2 and 3 of a 3-update trainer.run on 256 arena worlds x 8 robots."""
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.trainer import run
    sc = make_scenario('arena', robots_per_world=8, arenas=64, pick=1)
    env = StageWorld(512, scenario=sc, num_worlds=256, seed=0, auto_reset=0)
    policy = CNNPolicy(frames=3, action_space=2, seed=0, max_batch=max(1024, env.N))
    policy.load_state_dict(torch.load(STAGE2, map_location='cuda'))
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=128, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=1024, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=8, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    stats = run(env=env, policy=policy, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp,
                stage=2, max_updates=3, curriculum=CurriculumParams() if curriculum else None)
    return float(np.mean([s['agent_steps_per_s'] for s in stats[1:]]))


def main():
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info), flush=True)
    print('| launch | shape | case | us per call |')
    print('|---|---|---|---|')
    for K, W in ((8, 256), (16, 1024)):
        for (name, case), us in relayout_times(K, W).items():
            print('| %s | %d x %d | %s | %.1f |' % (name, W, K, case, us), flush=True)
    for T, us in update_times().items():
        print('| rlca_arena_curriculum_update | T = %d | | %.1f |' % (T, us), flush=True)
    rates = {}
    for _ in range(2):
        for cur in (False, True):
            rates.setdefault(cur, []).append(train_rate(cur))
    for cur in (False, True):
        print('trainer.run 256 x 8 arenas%s: agent-steps/s per pass %s' % (
            ' --arena-curriculum' if cur else '', ', '.join('%.0f' % r for r in rates[cur])), flush=True)


if __name__ == '__main__':
    main()
