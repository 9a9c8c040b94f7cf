#!/usr/bin/env python
"""Cost and shaping jumps of training with the global planner (DESIGN.md §9x), on the card named in the output (with its
power limit and maximum SM clock):
  - rlca_plan_shape (in place, after a tick) against rlca_plan_waypoints, CUDA events round 200 calls, two passes, at
    stage 1 171 x 24, stage 2 24 x 44 and arenas 1024 x 16;
  - trainer.run's rollout_s and agent-steps/s with and without the planner ('geodesic') at arenas 256 x 8, stage 1
    43 x 24 and stage 2 24 x 44 (mean of updates 2 and 3 of a 3-update run from stage2.pth);
  - on the arena run, |psi_prev - psi| of every non-terminal robot-tick: the share above 0.05 m and 0.2 m and the
    maximum, overall and per status transition, the largest jump's row, and the share of status-2 (no plan)
    robot-ticks.

    python tools/time_planner_train.py
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_collision_avoidance_b200 import planner as planner_mod  # noqa: E402
from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy  # noqa: E402
from rl_collision_avoidance_b200.planner import Planner  # noqa: E402
from rl_collision_avoidance_b200.scenarios import make_scenario  # noqa: E402
from rl_collision_avoidance_b200.stage_world import StageWorld  # noqa: E402
from rl_collision_avoidance_b200.trainer import run  # noqa: E402
from time_planner import events  # noqa: E402

STAGE2 = os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth')
AUTO_RESET = {'stage1': 1, 'stage2': 2, 'arena': 0}


def scenario(name, K=16, pick=0):
    return make_scenario('arena', robots_per_world=K, arenas=64, pick=pick) if name == 'arena' else make_scenario(name)


def launches():
    for name, W in (('stage1', 171), ('stage2', 24), ('arena', 1024)):
        sc = scenario(name)
        env = StageWorld(512, scenario=sc, num_worlds=W, seed=0, auto_reset=AUTO_RESET[name])
        env.reset_world()
        env.reset_pose()
        if sc.layout is not None:
            env.random_layout()
        p = Planner(env, reward=True)
        p.update()
        a = torch.rand(env.N, 2, device='cuda')
        env.control_vel(a, live=env.live if sc.layout is not None else None)
        p.update(env.flags)
        lib, cfg, st = env.lib, env.cfg, env._state_struct(env._cur)
        gs, rw, ep = env.gs.clone(), env.reward.clone(), env.eplog.clone()
        ptr = lambda t: C.c_void_p(t.data_ptr())
        wp = lambda: lib.rlca_plan_waypoints(C.byref(cfg), C.byref(p._t), C.byref(p._st), C.byref(st), ptr(env.gs),
                                             ptr(p.gs), env._stream())
        shape = lambda: lib.rlca_plan_shape(C.byref(cfg), C.byref(p._t), C.byref(p._st), ptr(p.psi_prev),
                                            ptr(p.psi_start), C.byref(st), ptr(env.flags), ptr(rw), ptr(ep), ptr(gs),
                                            ptr(gs), env._stream())
        for pas in range(2):
            t_wp, t_sh = events(wp, 200), events(shape, 200)
            print('%s %d x %d pass %d: waypoints %.1f us  shape (in place) %.1f us'
                  % (name, W, sc.robots_per_world, pas, 1e3 * t_wp, 1e3 * t_sh), flush=True)
        del p, env
        torch.cuda.empty_cache()


def train(name, W, planner, updates=3):
    sc = scenario(name, 8, pick=1) if name == 'arena' else scenario(name)
    env = StageWorld(512, scenario=sc, num_worlds=W, seed=0, auto_reset=AUTO_RESET[name])
    pol = CNNPolicy(frames=3, action_space=2, seed=0, max_batch=max(1024, env.N))
    pol.load_state_dict(torch.load(STAGE2, map_location='cuda'))
    opt = Adam(pol.parameters(), lr=5e-5)
    stage = 1 if name == 'stage1' else 2
    hp = dict(HORIZON=128, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=1024 if stage == 1 else 512, EPOCH=2 if stage == 1 else 4,
              COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1, NUM_ENV=sc.robots_per_world, OBS_SIZE=512, ACT_SIZE=2,
              LASER_HIST=3, MAX_EPISODES=5000)
    stats = run(env=env, policy=pol, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp,
                stage=stage, max_updates=updates, generator=torch.Generator(device='cuda').manual_seed(0),
                planner=planner)
    return stats


def jumps():
    """Wrap Planner.update on an arena training run and collect |psi_prev - psi| of the non-terminal rows, binned by the
    status transition (status before -> after the tick), and the largest jump's row."""
    d, orig = [], planner_mod.Planner.update

    def update(self, flags=None, reward=None, eplog=None, gs=None):
        before = self.psi_prev.clone() if self.reward else None
        s_before = self.status().clone()
        out = orig(self, flags, reward, eplog, gs)
        if flags is not None and before is not None:
            live = flags[:, 0] == 0
            d.append(((before - self.psi_prev).abs()[live], s_before[live], self.status()[live], before[live],
                      self.psi_prev[live], self.env.state['pose'][live, 3]))
        return out
    planner_mod.Planner.update = update
    try:
        stats = train('arena', 256, 'geodesic', updates=2)
    finally:
        planner_mod.Planner.update = orig
    x, s0, s1, pp, psi, pw = (torch.cat([r[k] for r in d]).cpu().numpy() for k in range(6))
    x = x.astype(np.float64)
    no_plan = np.mean([s['planner']['no_plan'] for s in stats])
    wp = np.mean([s['planner']['waypoint'] for s in stats])
    print('jumps, arena 256 x 8 training rollout (2 updates, %d non-terminal robot-ticks): |psi_prev - psi| > 0.05 m '
          '%.4f, > 0.2 m %.4f, max %.3f m, mean %.4f m; status shares: waypoint %.3f, no plan %.5f'
          % (len(x), (x > 0.05).mean(), (x > 0.2).mean(), x.max(), x.mean(), wp, no_plan), flush=True)
    for a in range(3):
        for b in range(3):
            m = (s0 == a) & (s1 == b)
            if m.any():
                print('  status %d -> %d: %d robot-ticks (%.4f), > 0.05 m %d, > 0.2 m %d, max %.3f m, mean %.4f m'
                      % (a, b, m.sum(), m.mean(), (x[m] > 0.05).sum(), (x[m] > 0.2).sum(), x[m].max(), x[m].mean()),
                      flush=True)
    k = int(np.argmax(x))
    print('  largest jump: status %d -> %d, psi_prev %.3f m, psi %.3f m, straight-line distance after %.3f m'
          % (s0[k], s1[k], pp[k], psi[k], pw[k]), flush=True)


def main():
    try:
        info = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                               '0'], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        info = 'unknown'
    print('card: %s, power limit, max SM clock: %s' % (torch.cuda.get_device_name(0), info), flush=True)
    launches()
    for name, W in (('arena', 256), ('stage1', 43), ('stage2', 24)):
        for planner in (None, 'geodesic'):
            s = train(name, W, planner)[1:]
            print('train %s %d worlds, planner %s: rollout_s %.3f, update_s %.3f, agent-steps/s %.0f'
                  % (name, W, planner, np.mean([x['rollout_s'] for x in s]), np.mean([x['update_s'] for x in s]),
                     np.mean([x['agent_steps_per_s'] for x in s])), flush=True)
            torch.cuda.empty_cache()
    jumps()


if __name__ == '__main__':
    main()
