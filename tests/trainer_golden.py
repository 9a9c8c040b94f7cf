"""The single-env trainer run pinned bit for bit: two stage-2 updates of `trainer.run` from `stage2.pth` on a stage-2 env
and on a random-layout env, recorded as SHA-256 digests of the parameters, the env state and the `Env` log lines,
plus the per-update episode counts, rewards and losses.  tests/golden/trainer_single_env.json holds the record of the
trainer before mixed runs existed (commit 4398f1c), so a single-env run is checked against that trainer, not against
the new code's own list path.  GPU only.  To write the record with another trainer module:

    python tests/trainer_golden.py --trainer-module rl_collision_avoidance_b200.trainer --out /tmp/trainer.json
"""
import argparse
import hashlib
import importlib
import json
import logging
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'trainer_single_env.json')
CASES = ('stage2', 'random')


def make_env(name, seed=4):
    from rl_collision_avoidance_b200.scenarios import make_scenario
    from rl_collision_avoidance_b200.stage_world import StageWorld
    from rl_collision_avoidance_b200.stage_world2 import StageWorld as Stage2World
    if name == 'stage2':
        return Stage2World(512, num_worlds=4, seed=seed, auto_reset=2)
    sc = make_scenario('random', robots_per_world=8, side=6.0, timeout=25)
    return StageWorld(512, scenario=sc, num_worlds=16, seed=seed, auto_reset=0)


class _Lines(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def record(run, name, seed=4, updates=2):
    """The record of `run` (a trainer.run) on case `name`: 2 updates, horizon 64, batch 128, 2 epochs."""
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    env = make_env(name, seed)
    policy = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=max(128, env.N))
    policy.load_state_dict(torch.load(os.path.join(ROOT, 'tests', 'golden', 'checkpoints', 'stage2.pth'),
                                      map_location='cuda'))
    opt = Adam(policy.parameters(), lr=5e-5)
    hp = dict(HORIZON=64, GAMMA=0.99, LAMDA=0.95, BATCH_SIZE=128, EPOCH=2, COEFF_ENTROPY=5e-4, CLIP_VALUE=0.1,
              NUM_ENV=env.num_env, OBS_SIZE=512, ACT_SIZE=2, LASER_HIST=3, MAX_EPISODES=5000)
    lg = logging.getLogger('trainer_golden_%s_%d' % (name, id(env)))
    lg.setLevel(logging.INFO)
    lg.propagate = False
    h = _Lines()
    lg.addHandler(h)
    gen = torch.Generator(device='cuda').manual_seed(seed)
    stats = run(env=env, policy=policy, policy_path=None, action_bound=[[0, -1], [1, 1]], optimizer=opt, hp=hp,
                logger=lg, logger_cal=None, stage=2, max_updates=updates, generator=gen)
    lg.removeHandler(h)
    torch.cuda.synchronize()
    return {'params': _digest(policy.flat),
            'state': {k: _digest(v) for k, v in env.state.items()},
            'log': hashlib.sha256('\n'.join(h.lines).encode()).hexdigest(),
            'log_lines': len(h.lines),
            'stats': [{'episodes': s['episodes'], 'mean_ep_reward': s['mean_ep_reward'],
                       'success_rate': s['success_rate'], 'losses': [float(x) for x in s['losses']]} for s in stats]}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--trainer-module', default='rl_collision_avoidance_b200.trainer')
    ap.add_argument('--out', default=GOLDEN)
    args = ap.parse_args(argv)
    sys.path.insert(0, ROOT)
    run = importlib.import_module(args.trainer_module).run
    out = {name: record(run, name) for name in CASES}
    with open(args.out, 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write('\n')
    print(json.dumps(out, sort_keys=True)[:400])


if __name__ == '__main__':
    main()
