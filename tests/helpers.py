"""Shared helpers for the parity tests: build a GPU StageWorld and its oracle twin."""
import numpy as np

from oracle.oracle import OracleWorld, OrcConfig
from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario


def make_pair(scenario='stage1', num_worlds=3, beams=512, auto_reset=True, seed=0, ctas_per_world=0,
              world_offset=0, raw_beams=None, gpu=True, robots_per_world=None, radius=None, max_reject=4096):
    """`robots_per_world` and `radius` reshape stage 1 / circle (make_scenario); `max_reject` is the spawn sampler's
    try budget."""
    sc = make_scenario(scenario, robots_per_world=robots_per_world, radius=radius)
    ocfg = fill_config(OrcConfig(), sc, num_worlds=num_worlds, beams=beams, raw_beams=raw_beams,
                       auto_reset=auto_reset, seed=seed, world_offset=world_offset, max_reject=max_reject)
    orc = OracleWorld(ocfg, sc.map.cells, sc.init_tab, sc.goal_tab)
    env = None
    if gpu:
        from rl_collision_avoidance_b200.stage_world import StageWorld
        env = StageWorld(beams, index=0, scenario=sc, num_worlds=num_worlds, seed=seed, auto_reset=auto_reset,
                         ctas_per_world=ctas_per_world, world_offset=world_offset, raw_beams=raw_beams,
                         max_reject=max_reject)
    return sc, env, orc


def random_actions(rng, n, wide=False):
    lo, hi = (-0.3, 1.3) if wide else (0.0, 1.0)
    a = np.stack([rng.uniform(lo, hi, n), rng.uniform(-1.3 if wide else -1.0, 1.3 if wide else 1.0, n)], 1)
    return a.astype(np.float32)


def assert_state_equal(env, orc, tag=''):
    import torch
    torch.cuda.synchronize()
    st = env.state
    for k, ref in (('pose', orc.pose), ('goal', orc.goal), ('acc', orc.acc), ('meta', orc.meta)):
        got = st[k].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), f'{tag}: state {k} differs at rows ' \
            f'{np.unique(np.nonzero(got.view(np.uint32) != ref.view(np.uint32))[0])[:8]}'


def assert_outputs_equal(env, orc, tag='', obs=None):
    import torch
    torch.cuda.synchronize()
    o = (env.obs if obs is None else obs).cpu().numpy()
    assert np.array_equal(o.view(np.uint32), orc.obs.view(np.uint32)), \
        f'{tag}: obs differ, max abs {np.abs(o - orc.obs).max()} at {np.argwhere(o != orc.obs)[:4]}'
    assert np.array_equal(env.gs.cpu().numpy().view(np.uint32), orc.gs.view(np.uint32)), f'{tag}: gs differ'
