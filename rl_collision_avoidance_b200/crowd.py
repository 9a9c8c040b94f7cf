"""A reactive crowd (DESIGN.md §9t): masked agents driven by a Helbing-Molnar style social-force controller on the
device (csrc/rlca_orca.cu, rlca_crowd_action).  Each crowd agent is drawn towards its goal at `speed`, repelled by the
other agents of its world (all of them, or with see_robots=False only the other crowd agents: the "invisible robot"
setting of crowd-navigation benchmarks) and, with a map, by the static map's boundary.  A crowd agent is an env agent
with the robot's footprint and kinematics: the lidar and the collision test see it as they see any robot.

    crowd = Crowd(env, non_cooperative_mask(R, W, k), CrowdParams(), obstacles=True)
    crowd.apply(action)                     # overwrites the masked rows of any controller's or policy's action

`crowd_host` runs the same code on the CPU from numpy arrays and equals the kernel bit for bit.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import asdict, dataclass

import numpy as np
import torch

from . import _lib
from .orca import ObstacleSet, _ptr


@dataclass(frozen=True)
class CrowdParams:
    """The social-force parameters (DESIGN.md §9t): starting values in the range the social-force literature uses, not
    tuned ones.  speed None is cfg.v_max.  ValueError for a value the kernel refuses; speed against v_max and wall_dist
    against the obstacle set's range are checked where those are known (Crowd, crowd_host)."""
    speed: float = None             # m/s, in (0, v_max]
    relax_time: float = 0.5         # s
    strength: float = 5.0           # m/s^2 (2.0 and a 0.3 m range crash the K = 2 head-on pair: DESIGN.md §9t)
    range: float = 0.5              # m
    anisotropy: float = 0.35        # lambda in [0, 1]: the weight of a neighbour straight behind
    side_bias: float = 0.2          # share of the repulsion turned to the agent's right of the neighbour
    radius: float = 0.35            # m, ORCA-DD's
    neighbour_dist: float = 3.0     # m
    wall_strength: float = 5.0      # m/s^2
    wall_range: float = 0.1         # m
    wall_dist: float = 1.0          # m
    heading_gain: float = 2.0       # 1/s, the §9h driver's
    see_robots: bool = True

    def __post_init__(self):
        def fin(k):
            v = getattr(self, k)
            if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)):
                raise ValueError(f'crowd {k} must be a number, got {v!r}')
            return float(v)
        if self.speed is not None and not (math.isfinite(fin('speed')) and fin('speed') > 0.0):
            raise ValueError(f'crowd speed must be finite and > 0, got {self.speed!r}')
        for k in ('relax_time', 'range', 'wall_range', 'radius', 'neighbour_dist', 'heading_gain', 'wall_dist'):
            if not (math.isfinite(fin(k)) and fin(k) > 0.0):
                raise ValueError(f'crowd {k} must be finite and > 0, got {getattr(self, k)!r}')
        for k in ('strength', 'wall_strength', 'side_bias'):
            if not (math.isfinite(fin(k)) and fin(k) >= 0.0):
                raise ValueError(f'crowd {k} must be finite and >= 0, got {getattr(self, k)!r}')
        if not 0.0 <= fin('anisotropy') <= 1.0:
            raise ValueError(f'crowd anisotropy must be in [0, 1], got {self.anisotropy!r}')

    def struct(self, v_max):
        """The rlca_crowd_params of these settings; speed None becomes v_max."""
        d = asdict(self)
        d['speed'] = float(v_max) if self.speed is None else float(self.speed)
        d['see_robots'] = int(bool(self.see_robots))
        return _lib.CrowdParams(**d)


class Crowd:
    """Crowd agents (rlca_crowd_action): the agents with `mask` != 0 (N, held on the env's device as uint8) follow the
    social force of `params`.  `obstacles`: None / False is map-blind, True builds an ObstacleSet of env.sc.map with
    max_range = wall_dist, or an ObstacleSet (max_range >= wall_dist) to share."""

    def __init__(self, env, mask, params=None, obstacles=None):
        self.env = env
        self.params = CrowdParams() if params is None else params
        self.mask = torch.as_tensor(mask, device=env.device).to(torch.uint8).contiguous()
        if self.mask.shape != (env.N,):
            raise ValueError(f'mask must have ({env.N},) entries')
        speed = self.params.speed
        if speed is not None and not np.float32(speed) <= np.float32(env.cfg.v_max):
            raise ValueError(f'crowd speed must be in (0, {env.cfg.v_max:g}], got {speed!r}')
        if obstacles is True:
            with torch.cuda.device(env.device):
                obstacles = ObstacleSet(env.cfg, env.sc.map.cells, self.params.wall_dist)
        self.obstacles = obstacles or None
        if self.obstacles is not None and not self.params.wall_dist <= self.obstacles.max_range:
            raise ValueError('crowd wall_dist %g exceeds the obstacle set\'s max_range %g'
                             % (self.params.wall_dist, self.obstacles.max_range))
        self._p = self.params.struct(env.cfg.v_max)

    def apply(self, action):
        """Overwrite the masked rows of `action` ((N, 2) float32, contiguous, on the env's device) in place, from the
        state the next tick reads, on the env's stream; returns `action`."""
        env = self.env
        if action.shape != (env.N, 2) or action.dtype != torch.float32 or not action.is_contiguous() or \
                action.device != self.mask.device:
            raise ValueError(f'action must be a contiguous ({env.N}, 2) float32 tensor on {self.mask.device}')
        st = env._state_struct(env._cur)
        obs = self.obstacles.handle if self.obstacles is not None else None
        _lib.check(env.lib.rlca_crowd_action(C.byref(env.cfg), C.byref(self._p), C.byref(st), _ptr(self.mask), obs,
                                             _ptr(action), env._stream()))
        return action

    def settings(self):
        d = asdict(self.params)
        d['speed'] = float(self._p.speed)
        d['map'] = self.obstacles is not None
        d['agents'] = int(self.mask.count_nonzero())
        return d


def crowd_host(cfg, pose, goal, meta, mask, action, params=None, obstacles=None):
    """rlca_crowd_action_host on numpy arrays (pose, goal (N, 4) float32, meta (N, 4) int32, mask (N) uint8): returns a
    copy of `action` (N, 2) whose rows with mask != 0 are overwritten.  `obstacles`: None (map-blind) or an
    ObstacleSet."""
    lib = _lib.load()
    params = CrowdParams() if params is None else params
    p = np.ascontiguousarray(pose, np.float32)
    g = np.ascontiguousarray(goal, np.float32)
    m = np.ascontiguousarray(meta, np.int32)
    k = np.ascontiguousarray(mask, np.uint8)
    act = np.array(action, np.float32, order='C', copy=True)
    n = cfg.robots_per_world * cfg.num_worlds
    if p.shape != (n, 4) or g.shape != (n, 4) or m.shape != (n, 4) or k.shape != (n,) or act.shape != (n, 2):
        raise ValueError(f'pose, goal and meta must be ({n}, 4), mask ({n},) and action ({n}, 2)')
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    ps = params.struct(cfg.v_max)
    _lib.check(lib.rlca_crowd_action_host(C.byref(cfg), C.byref(ps), obstacles.handle if obstacles else None, vp(p),
                                          vp(g), vp(m), vp(k), vp(act)))
    return act


# ------------------------------------------------------------------------------------------------ command line
CROWD_FLAGS = ('--crowd-speed', '--crowd-ignores-robots', '--crowd-map', '--crowd-strength', '--crowd-range',
               '--crowd-side-bias')


def add_crowd_arguments(ap, non_cooperative=False):
    """The crowd flags of a driver on an argparse parser; with non_cooperative also --non-cooperative K and
    --non-cooperative-speed (the trainers; evaluate.py has its own)."""
    d = CrowdParams()
    if non_cooperative:
        ap.add_argument('--non-cooperative', type=int, default=None, metavar='K',
                        help='K robots of every world drive straight to their goals, ignoring everyone (DESIGN.md '
                             '§9h); their rows are left out of every PPO update')
        ap.add_argument('--non-cooperative-speed', type=float, default=None, metavar='S',
                        help='speed of the non-cooperative robots, m/s, in (0, v_max] (default v_max)')
    ap.add_argument('--crowd', type=int, default=None, metavar='K',
                    help='K agents of every world are a social-force crowd (DESIGN.md §9t)')
    ap.add_argument('--crowd-speed', type=float, default=None, metavar='S',
                    help='preferred speed of the crowd, m/s, in (0, v_max] (default v_max)')
    ap.add_argument('--crowd-ignores-robots', action='store_true',
                    help='the crowd avoids only itself and the map, not the other agents')
    ap.add_argument('--crowd-map', action='store_true', help='the crowd also avoids the static map')
    ap.add_argument('--crowd-strength', type=float, default=None, metavar='A',
                    help='agent repulsion strength, m/s^2, >= 0 (default %g)' % d.strength)
    ap.add_argument('--crowd-range', type=float, default=None, metavar='B',
                    help='agent repulsion range, m, > 0 (default %g)' % d.range)
    ap.add_argument('--crowd-side-bias', type=float, default=None, metavar='C',
                    help='sideways share of the agent repulsion, >= 0 (default %g)' % d.side_bias)


def crowd_from_arguments(ap, args, v_max, robots_per_world=None):
    """(k, CrowdParams, map flag) of the crowd flags, or None without --crowd; ap.error for a crowd flag without
    --crowd, --crowd with --non-cooperative, k outside 1..robots_per_world (when given) and a bad value."""
    if args.crowd is None:
        given = [f for f in CROWD_FLAGS if getattr(args, f[2:].replace('-', '_')) not in (None, False)]
        if given:
            ap.error('%s applies with --crowd only' % given[0])
        return None
    if getattr(args, 'non_cooperative', None) is not None:
        ap.error('--crowd and --non-cooperative cannot be combined: the metrics split into two roles')
    if args.crowd < 1 or (robots_per_world is not None and args.crowd > robots_per_world):
        ap.error('--crowd must be in 1..%s' % (robots_per_world if robots_per_world is not None else 'R'))
    if args.crowd_speed is not None and not 0.0 < args.crowd_speed <= v_max:
        ap.error('--crowd-speed must be in (0, %g]' % v_max)
    kw = {k: getattr(args, 'crowd_' + k) for k in ('speed', 'strength', 'range', 'side_bias')
          if getattr(args, 'crowd_' + k) is not None}
    try:
        params = CrowdParams(see_robots=not args.crowd_ignores_robots, **kw)
    except ValueError as e:
        ap.error('--crowd: %s' % e)
    return args.crowd, params, bool(args.crowd_map)


def non_cooperative_from_arguments(ap, args, v_max):
    """(k, speed) of the trainers' --non-cooperative flags, or None; ap.error for a bad value.  k against the robots of
    a world is checked when the envs exist (trainer.run: ValueError)."""
    if args.non_cooperative is None:
        if args.non_cooperative_speed is not None:
            ap.error('--non-cooperative-speed applies with --non-cooperative only')
        return None
    if args.non_cooperative < 1:
        ap.error('--non-cooperative must be >= 1')
    if args.non_cooperative_speed is not None and not 0.0 < args.non_cooperative_speed <= v_max:
        ap.error('--non-cooperative-speed must be in (0, %g]' % v_max)
    return args.non_cooperative, args.non_cooperative_speed
