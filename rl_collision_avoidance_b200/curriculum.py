"""Automatic curriculum over generated arenas (DESIGN.md §9z): per-arena episode outcomes tallied on the device, and
re-layouts that draw a world's arena in proportion to how much the policy can still learn there.

Per arena a the curriculum keeps decayed episode and success counts E_a, S_a (float32).  After each tick the weighted
re-layout launch (rlca_layout_arena_weighted_respawn, in place of pick 1's rlca_layout_arena_respawn) adds the tick's
ended, unmasked rows of every world to the integer counts of the arena the world is in.  Once per PPO update
rlca_arena_curriculum_update folds them in, E_a = decay E_a + e_a, S_a = decay S_a + s_a, and scores the arena by its
learnability p (1 - p), p = (S_a + 1) / (E_a + 2) (a Laplace prior: an arena without recent episodes scores p = 1/2,
the highest), mixed with a uniform floor: q_a = uniform + (1 - uniform) 4 p (1 - p).  A world's next arena is drawn
in proportion to the integer weights w_a = max(1, floor(2^20 q_a)).  With all weights equal (at the start) the draw is
pick 1's, bit for bit.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .scenarios import ArenaLayout, arena_tables_struct


@dataclass(frozen=True)
class CurriculumParams:
    """decay: the weight of the counts before an update, in [0, 1); uniform: the share of every arena's score that does
    not depend on its outcomes, in [0, 1] (1 draws every arena equally often, as pick 1 does).  The defaults are
    untuned."""
    decay: float = 0.9
    uniform: float = 0.1


def check_params(params):
    """`params` with float32 values; ValueError for decay outside [0, 1) or uniform outside [0, 1], NaN included."""
    d, u = float(np.float32(params.decay)), float(np.float32(params.uniform))
    if not 0.0 <= d < 1.0:
        raise ValueError(f'curriculum decay must be in [0, 1), got {params.decay}')
    if not 0.0 <= u <= 1.0:
        raise ValueError(f'curriculum uniform must be in [0, 1], got {params.uniform}')
    return CurriculumParams(d, u)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class ArenaCurriculum:
    """The curriculum of one arena env (stage_world.StageWorld on an arena scenario with pick 1): its device buffers,
    attached to the env, whose random_layout() and relayout_finished() then draw arenas by the curriculum's weights.
    `row_mask` (N,) marks the rows whose episodes are not counted (masked agents), None counts every row."""

    def __init__(self, env, params=CurriculumParams(), row_mask=None):
        lay = env.sc.layout
        if not isinstance(lay, ArenaLayout):
            raise ValueError(f'an arena curriculum needs an arena scenario, got {env.sc.name}')
        if lay.pick != 1:
            raise ValueError(f'an arena curriculum replaces the arena draw of pick 1 (training); the scenario has pick '
                             f'{lay.pick}')
        self.params = check_params(params)
        self.env = env
        self.T = lay.count
        self.arena_seed = int(lay.seed)
        dev = env.device
        self.cdf = torch.zeros(self.T + 1, dtype=torch.int64, device=dev)        # uint64 values, all < 2^63
        self.world_arena = torch.zeros(env.num_worlds, dtype=torch.int32, device=dev)
        self.pending = torch.zeros(2 * self.T, dtype=torch.int32, device=dev)
        self.E = torch.zeros(self.T, dtype=torch.float32, device=dev)
        self.S = torch.zeros(self.T, dtype=torch.float32, device=dev)
        self.row_mask = None
        if row_mask is not None:
            m = torch.as_tensor(np.asarray(row_mask) != 0).to(device=dev, dtype=torch.uint8).contiguous()
            if m.shape != (env.N,):
                raise ValueError(f'row_mask must have {env.N} rows, got shape {tuple(m.shape)}')
            self.row_mask = m
        self.struct = _lib.ArenaCurriculum(self.T, _ptr(self.cdf), _ptr(self.world_arena), _ptr(self.pending),
                                           _ptr(self.E), _ptr(self.S))
        self.folded = torch.zeros((), dtype=torch.int64, device=dev)
        self._fold()                                     # E = S = 0: equal weights
        env.curriculum = self

    def _fold(self):
        _lib.check(self.env.lib.rlca_arena_curriculum_update(C.byref(self.struct), self.params.decay,
                                                             self.params.uniform, self.env._stream()))

    def update(self, process_group=None):
        """Fold the counts tallied since the last update into E and S and draw from the new weights.  Under data
        parallelism (`process_group` a group, or True for the default one) the counts are first summed over the ranks
        (one all-reduce of 2 T int32), so every rank holds the same weights."""
        if process_group is not None:
            import torch.distributed as dist
            dist.all_reduce(self.pending, group=None if process_group is True else process_group)
        self.folded = self.pending[:self.T].sum()
        self._fold()

    def weights(self):
        """(T,) int64 weights of the next draws (one synchronisation)."""
        return np.diff(self.cdf.cpu().numpy())

    def stats(self):
        """The effective number of arenas exp(H) of the draw distribution w / sum(w), its largest and smallest share,
        and the episodes folded in at the last update."""
        w = self.weights().astype(np.float64)
        share = w / w.sum()
        return {'arenas': self.T, 'effective_arenas': float(math.exp(-(share * np.log(share)).sum())),
                'max_share': float(share.max()), 'min_share': float(share.min()), 'episodes': int(self.folded)}

    def state_dict(self):
        return {'num_arenas': self.T, 'arena_seed': self.arena_seed, 'decay': self.params.decay,
                'uniform': self.params.uniform, 'E': self.E.cpu(), 'S': self.S.cpu(), 'cdf': self.cdf.cpu(),
                'pending': self.pending.cpu()}

    def load_state_dict(self, sd):
        """Restore E, S, the weights and the pending counts.  ValueError for another arena count or arena seed."""
        if int(sd['num_arenas']) != self.T:
            raise ValueError(f'curriculum state holds {int(sd["num_arenas"])} arenas, the scenario has {self.T}')
        if int(sd['arena_seed']) != self.arena_seed:
            raise ValueError(f'curriculum state is for arena seed {int(sd["arena_seed"])}, the scenario has '
                             f'{self.arena_seed}')
        for name in ('E', 'S', 'cdf', 'pending'):
            dst, src = getattr(self, name), sd[name]
            if tuple(src.shape) != tuple(dst.shape) or src.dtype != dst.dtype:
                raise ValueError(f'curriculum state: {name} is {tuple(src.shape)} {src.dtype}, expected '
                                 f'{tuple(dst.shape)} {dst.dtype}')
            dst.copy_(src)


# ---------------------------------------------------------------------------------------------- host twins
def _host_struct(T, cdf, world_arena, pending, E, S):
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    return _lib.ArenaCurriculum(T, vp(cdf), vp(world_arena), vp(pending), vp(E), vp(S))


def update_host(E, S, pending, decay, uniform):
    """rlca_arena_curriculum_update_host on copies: (E, S, pending (zeroed), cdf (T + 1,) uint64)."""
    E, S = (np.array(a, np.float32, order='C', copy=True) for a in (E, S))
    pending = np.array(pending, np.int32, order='C', copy=True)
    T = len(E)
    cdf = np.zeros(T + 1, np.uint64)
    st = _host_struct(T, cdf, np.zeros(1, np.int32), pending, E, S)
    _lib.check(_lib.load().rlca_arena_curriculum_update_host(C.byref(st), float(decay), float(uniform)))
    return E, S, pending, cdf


def layout_host(cfg, layout, cdf, world_arena, pose, goal, acc):
    """rlca_layout_arena_weighted_host on copies: (pose, goal, acc, status, world_arena)."""
    lib = _lib.load()
    pose, goal, acc = (np.array(a, np.float32, order='C', copy=True) for a in (pose, goal, acc))
    cdf = np.ascontiguousarray(cdf, np.uint64)
    world_arena = np.array(world_arena, np.int32, order='C', copy=True)
    T = len(cdf) - 1
    status = np.full(int(cfg.num_worlds), -1, np.int32)
    st = _host_struct(T, cdf, world_arena, np.zeros(2 * T, np.int32), np.zeros(T, np.float32), np.zeros(T, np.float32))
    params = _lib.LayoutParams(layout.side, layout.separation, layout.min_travel)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_layout_arena_weighted_host(C.byref(cfg), C.byref(params), C.byref(arena_tables_struct(
        layout.tables)), C.byref(st), vp(pose), vp(goal), vp(acc), vp(status)))
    return pose, goal, acc, status, world_arena


def relayout_host(cfg, layout, cdf, world_arena, pending, row_mask, pose, goal, acc, meta, flags):
    """rlca_layout_arena_weighted_respawn_host on copies: (pose, goal, acc, meta, flags, live, status, world_arena,
    pending).  row_mask None counts every row."""
    lib = _lib.load()
    pose, goal, acc = (np.array(a, np.float32, order='C', copy=True) for a in (pose, goal, acc))
    meta = np.array(meta, np.int32, order='C', copy=True)
    flags = np.array(flags, np.uint8, order='C', copy=True)
    cdf = np.ascontiguousarray(cdf, np.uint64)
    world_arena = np.array(world_arena, np.int32, order='C', copy=True)
    pending = np.array(pending, np.int32, order='C', copy=True)
    T = len(cdf) - 1
    n = int(cfg.robots_per_world) * int(cfg.num_worlds)
    live = np.full(n, 0xFF, np.uint8)
    status = np.full(int(cfg.num_worlds), -1, np.int32)
    mask = None if row_mask is None else np.ascontiguousarray(np.asarray(row_mask) != 0, np.uint8)
    st = _host_struct(T, cdf, world_arena, pending, np.zeros(T, np.float32), np.zeros(T, np.float32))
    params = _lib.LayoutParams(layout.side, layout.separation, layout.min_travel)
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    _lib.check(lib.rlca_layout_arena_weighted_respawn_host(
        C.byref(cfg), C.byref(params), C.byref(arena_tables_struct(layout.tables)), C.byref(st), vp(mask), vp(pose),
        vp(goal), vp(acc), vp(meta), vp(flags), vp(live), vp(status)))
    return pose, goal, acc, meta, flags, live, status, world_arena, pending
