"""Scenario definitions: constants of the reference's three environments and the
spawn/goal tables, as data for the simulator kernels.

Sources (under /root/reference): stage_world1.py, stage_world2.py,
circle_world.py (rewards, thresholds, timeouts), worlds/*.world (geometry),
model/utils.py:6-63 (tables; shipped here as assets/scenarios.json produced by
tools/build_assets.py).  SURVEY.md Appendix B lists every constant.
"""
from __future__ import annotations

import dataclasses
import json
import math
import os
from dataclasses import dataclass

import numpy as np

from .worldfile import WorldMap, load_map

ASSETS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'assets')


@dataclass(frozen=True)
class Layout:
    """Parameters of a random layout (rlca_layout_params, DESIGN.md §9i), in metres."""
    side: float                # starts and goals lie in the square [-side/2, side/2]^2
    separation: float          # least start-start and goal-goal distance
    min_travel: float          # least start-goal distance


@dataclass(frozen=True, eq=False)
class ArenaLayout:
    """Parameters of an arena layout (rlca_layout_arena, DESIGN.md §9v): every world lays its robots out in one arena of
    a generated map (arenas.generate_arenas), in metres."""
    separation: float          # least start-start and goal-goal distance
    min_travel: float          # least start-goal distance
    pick: int                  # 0: world w in arena (world_offset + w) mod T; 1: an arena drawn at every layout
    tables: object             # arenas.ArenaTables of the map
    count: int                 # the generator's arguments
    side: float
    obstacles: tuple
    seed: int


@dataclass
class Scenario:
    name: str
    scenario_id: int           # 0 stage1, 1 stage2, 2 circle
    robots_per_world: int
    timeout: int
    w_threshold: float
    pre_distance_zero: int
    map: WorldMap
    init_tab: np.ndarray       # (R,4) x,y,theta,random_flag  float32
    goal_tab: np.ndarray       # (R,4) gx,gy,random_flag,group id   float32
    groups: tuple = ()         # stage-2 group boundaries (model/utils.py:83)
    layout: Layout | ArenaLayout | None = None   # random / arena scenario: every world draws its own layout
                                                 # (StageWorld.random_layout)


# constants shared by the three env clients (stage_world1.py:34,183-204)
COMMON = dict(dt=0.1, range_max=6.0, fov=math.pi, raw_beams=512, half_len=0.22, half_wid=0.19,
              goal_radius=0.5, reward_arrive=15.0, reward_collision=-15.0, progress_gain=2.5,
              w_penalty=-0.1, v_min=0.0, v_max=1.0, w_min=-1.0, w_max=1.0)


def _tables():
    with open(os.path.join(ASSETS, 'scenarios.json')) as f:
        return json.load(f)


def _footprint_cells(sc_map: WorldMap, x, y, th):
    """(K, P) cell rows, cols covering the footprint rectangles at poses (x, y, th): points every half cell over the
    rectangle, edges included, in the kernels' cell convention cell = floor(coord * ppm) + origin."""
    hl, hw = COMMON['half_len'], COMMON['half_wid']
    step = 0.5 * sc_map.resolution
    u = np.linspace(-hl, hl, int(math.ceil(2 * hl / step)) + 1)
    v = np.linspace(-hw, hw, int(math.ceil(2 * hw / step)) + 1)
    uu, vv = (a.ravel() for a in np.meshgrid(u, v))
    c, s = np.cos(th)[:, None], np.sin(th)[:, None]
    px = x[:, None] + c * uu - s * vv
    py = y[:, None] + s * uu + c * vv
    ppm = 1.0 / sc_map.resolution
    return np.floor(py * ppm).astype(np.int64) + sc_map.origin_cy, np.floor(px * ppm).astype(np.int64) + sc_map.origin_cx


def _rects_overlap(p, q):
    """Separating-axis test of two footprint rectangles given as (x, y, theta); touching counts as overlapping."""
    hl, hw = COMMON['half_len'], COMMON['half_wid']
    corners = []
    for x, y, th in (p, q):
        c, s = math.cos(th), math.sin(th)
        corners.append([(x + c * a - s * b, y + s * a + c * b) for a, b in ((hl, hw), (-hl, hw), (-hl, -hw), (hl, -hw))])
    for th in (p[2], q[2]):
        for ax in ((math.cos(th), math.sin(th)), (-math.sin(th), math.cos(th))):
            pa = [cx * ax[0] + cy * ax[1] for cx, cy in corners[0]]
            pb = [cx * ax[0] + cy * ax[1] for cx, cy in corners[1]]
            if max(pa) < min(pb) or max(pb) < min(pa):
                return False
    return True


def circle_layout(m: WorldMap, robots: int, radius: float):
    """(init_tab, goal_tab) of `robots` robots on a circle of `radius` metres: robot i at r (cos 2 pi i/K, sin 2 pi i/K)
    facing the centre (heading pi + 2 pi i/K wrapped to (-pi, pi]), its goal the antipode.  ValueError when K is
    outside 2..RLCA_MAX_ROBOTS_PER_WORLD, a start footprint covers a non-free or off-map cell, or neighbouring start
    footprints overlap."""
    K = int(robots)
    if not 2 <= K <= 64:
        raise ValueError(f'circle: robots_per_world must be in 2..64, got {robots}')
    r = float(radius)
    if not r > 0:
        raise ValueError(f'circle: radius must be > 0, got {radius}')
    a = 2.0 * np.pi * np.arange(K) / K
    x, y = r * np.cos(a), r * np.sin(a)
    th = np.remainder(np.pi + a + np.pi, 2.0 * np.pi) - np.pi
    th = np.where(th <= -np.pi, th + 2.0 * np.pi, th)
    rows, cols = _footprint_cells(m, x, y, th)
    inside = (rows >= 0) & (rows < m.grid_h) & (cols >= 0) & (cols < m.grid_w)
    free = inside.copy()
    free[inside] = m.cells[rows[inside], cols[inside]] == 0
    bad = np.nonzero(~free.all(1))[0]
    if len(bad):
        raise ValueError(f'circle: the start footprint of robot {bad[0]} (K={K}, r={r}) is not in free cells')
    for i in range(K):
        j = (i + 1) % K
        if i != j and _rects_overlap((x[i], y[i], th[i]), (x[j], y[j], th[j])):
            raise ValueError(f'circle: start footprints of robots {i} and {j} overlap (K={K}, r={r})')
    init = np.zeros((K, 4), np.float32)
    init[:, 0], init[:, 1], init[:, 2] = x, y, th
    goal = np.zeros((K, 4), np.float32)
    goal[:, 0], goal[:, 1] = -x, -y
    return init, goal


RANDOM_DEFAULTS = dict(robots_per_world=8, side=10.0, separation=1.0)     # min_travel defaults to side / 2


def _check_separation(who, resolution, D, separation):
    """(r_c, resolution) in the float32 values rlca_layout_random reads; ValueError for a separation it rejects."""
    hl, hw = (float(np.float32(COMMON[k])) for k in ('half_len', 'half_wid'))
    res = float(np.float32(resolution))
    rc = math.sqrt(hl * hl + hw * hw)
    d_min = 2.0 * (rc + math.sqrt(2.0) * res)
    if not (math.isfinite(D) and D > d_min):
        raise ValueError(f'{who}: separation must be finite and > {d_min:.4g} m (two footprints closer than that can '
                         f'share a cell), got {separation}')
    return rc, res


def random_layout_params(m: WorldMap, robots: int, side: float, separation: float, min_travel: float) -> Layout:
    """The Layout of a random scenario on map `m` after the checks rlca_layout_random makes (in float32, as it sees the
    values), and that the square grown by the footprint's circumradius r_c and one cell lies on free cells of the map.
    ValueError otherwise."""
    K = int(robots)
    if not 2 <= K <= 64:
        raise ValueError(f'random: robots_per_world must be in 2..64, got {robots}')
    S, D, L = (float(np.float32(v)) for v in (side, separation, min_travel))
    if not (math.isfinite(S) and S > 0):
        raise ValueError(f'random: side must be finite and > 0, got {side}')
    if not 0 <= L <= S * math.sqrt(2.0):
        raise ValueError(f'random: min_travel must be in [0, side * sqrt(2)] = [0, {S * math.sqrt(2.0):.4g}], '
                         f'got {min_travel}')
    rc, res = _check_separation('random', m.resolution, D, separation)
    e = 0.5 * S + rc + res
    ppm = 1.0 / m.resolution
    c0, c1 = math.floor(-e * ppm) + m.origin_cx, math.floor(e * ppm) + m.origin_cx
    r0, r1 = math.floor(-e * ppm) + m.origin_cy, math.floor(e * ppm) + m.origin_cy
    if c0 < 0 or r0 < 0 or c1 >= m.grid_w or r1 >= m.grid_h or m.cells[r0:r1 + 1, c0:c1 + 1].any():
        raise ValueError(f'random: the {S:g} m square grown by {rc + res:.3f} m is not on free cells of the map')
    return Layout(S, D, L)


def random_layout_host(cfg, layout: Layout, pose, goal, acc):
    """rlca_layout_random_host: the layout of every world of `cfg` (an EnvConfig) written into copies of the host
    arrays pose, goal, acc (N, 4) float32.  Returns (pose, goal, acc, status (num_worlds,) int32: 0 placed, 1 + r when
    robot r was not)."""
    import ctypes as C
    from . import _lib
    lib = _lib.load()
    pose, goal, acc = (np.array(a, np.float32, order='C', copy=True) for a in (pose, goal, acc))
    n = int(cfg.robots_per_world) * int(cfg.num_worlds)
    if any(a.shape != (n, 4) for a in (pose, goal, acc)):
        raise ValueError(f'pose, goal and acc must be ({n}, 4)')
    status = np.full(int(cfg.num_worlds), -1, np.int32)
    params = _lib.LayoutParams(layout.side, layout.separation, layout.min_travel)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_layout_random_host(C.byref(cfg), C.byref(params), vp(pose), vp(goal), vp(acc), vp(status)))
    return pose, goal, acc, status


def relayout_host(cfg, layout: Layout, pose, goal, acc, meta, flags):
    """rlca_layout_respawn_host (DESIGN.md §9k): the parking and re-layout after a tick of an env with auto_reset 0,
    written into copies of the host arrays pose, goal, acc (N, 4) float32, meta (N, 4) int32 and flags (N, 4) uint8.
    Returns (pose, goal, acc, meta, flags, live (N,) uint8, status (num_worlds,) int32)."""
    import ctypes as C
    from . import _lib
    lib = _lib.load()
    pose, goal, acc = (np.array(a, np.float32, order='C', copy=True) for a in (pose, goal, acc))
    meta = np.array(meta, np.int32, order='C', copy=True)
    flags = np.array(flags, np.uint8, order='C', copy=True)
    n = int(cfg.robots_per_world) * int(cfg.num_worlds)
    if any(a.shape != (n, 4) for a in (pose, goal, acc, meta, flags)):
        raise ValueError(f'pose, goal, acc, meta and flags must be ({n}, 4)')
    live = np.full(n, 0xFF, np.uint8)
    status = np.full(int(cfg.num_worlds), -1, np.int32)
    params = _lib.LayoutParams(layout.side, layout.separation, layout.min_travel)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_layout_respawn_host(C.byref(cfg), C.byref(params), vp(pose), vp(goal), vp(acc), vp(meta),
                                            vp(flags), vp(live), vp(status)))
    return pose, goal, acc, meta, flags, live, status


def arena_tables_struct(tables, cell_off_ptr=None, cells_ptr=None):
    """The rlca_arena_tables of `tables` (arenas.ArenaTables): host pointers into its arrays, or the given device
    pointers."""
    from . import _lib
    if cell_off_ptr is None:
        cell_off_ptr, cells_ptr = tables.cell_off.ctypes.data, tables.cells.ctypes.data
    return _lib.ArenaTables(tables.count, cell_off_ptr, cells_ptr)


def arena_layout_host(cfg, layout: ArenaLayout, pose, goal, acc, pick=None):
    """rlca_layout_arena_host: the arena layout of every world of `cfg` written into copies of the host arrays pose,
    goal, acc (N, 4) float32; `pick` overrides the layout's.  Returns (pose, goal, acc, status (num_worlds,) int32)."""
    import ctypes as C
    from . import _lib
    lib = _lib.load()
    pose, goal, acc = (np.array(a, np.float32, order='C', copy=True) for a in (pose, goal, acc))
    n = int(cfg.robots_per_world) * int(cfg.num_worlds)
    if any(a.shape != (n, 4) for a in (pose, goal, acc)):
        raise ValueError(f'pose, goal and acc must be ({n}, 4)')
    status = np.full(int(cfg.num_worlds), -1, np.int32)
    params = _lib.LayoutParams(layout.side, layout.separation, layout.min_travel)
    tab = arena_tables_struct(layout.tables)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_layout_arena_host(C.byref(cfg), C.byref(params), C.byref(tab),
                                          layout.pick if pick is None else pick, vp(pose), vp(goal), vp(acc),
                                          vp(status)))
    return pose, goal, acc, status


def arena_relayout_host(cfg, layout: ArenaLayout, pose, goal, acc, meta, flags, pick=None):
    """rlca_layout_arena_respawn_host: relayout_host with the arena sampler.  Returns (pose, goal, acc, meta, flags,
    live (N,) uint8, status (num_worlds,) int32)."""
    import ctypes as C
    from . import _lib
    lib = _lib.load()
    pose, goal, acc = (np.array(a, np.float32, order='C', copy=True) for a in (pose, goal, acc))
    meta = np.array(meta, np.int32, order='C', copy=True)
    flags = np.array(flags, np.uint8, order='C', copy=True)
    n = int(cfg.robots_per_world) * int(cfg.num_worlds)
    if any(a.shape != (n, 4) for a in (pose, goal, acc, meta, flags)):
        raise ValueError(f'pose, goal, acc, meta and flags must be ({n}, 4)')
    live = np.full(n, 0xFF, np.uint8)
    status = np.full(int(cfg.num_worlds), -1, np.int32)
    params = _lib.LayoutParams(layout.side, layout.separation, layout.min_travel)
    tab = arena_tables_struct(layout.tables)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_layout_arena_respawn_host(C.byref(cfg), C.byref(params), C.byref(tab),
                                                  layout.pick if pick is None else pick, vp(pose), vp(goal), vp(acc),
                                                  vp(meta), vp(flags), vp(live), vp(status)))
    return pose, goal, acc, meta, flags, live, status


def random_max_ticks(side):
    """3 x the ticks the square's diagonal takes at v_max: the default tick budget of a random scenario, for an
    evaluation run and for a training episode alike."""
    return 3 * math.ceil(side * math.sqrt(2.0) / (COMMON['v_max'] * COMMON['dt']))


RANDOM_FLAGS = ('--random-robots', '--random-side', '--random-separation', '--random-min-travel')


def add_random_arguments(ap, timeout=False):
    """The --random-* flags of a random scenario on an argparse parser; `timeout` adds --random-timeout (training)."""
    ap.add_argument('--random-robots', type=int, default=None, metavar='K',
                    help='random: robots per world, 2..64 (default %d)' % RANDOM_DEFAULTS['robots_per_world'])
    ap.add_argument('--random-side', type=float, default=None, metavar='S',
                    help='random: side of the square of starts and goals, m (default %g)' % RANDOM_DEFAULTS['side'])
    ap.add_argument('--random-separation', type=float, default=None, metavar='D',
                    help='random: least start-start and goal-goal distance, m (default %g)'
                         % RANDOM_DEFAULTS['separation'])
    ap.add_argument('--random-min-travel', type=float, default=None, metavar='L',
                    help='random: least start-goal distance, m (default S / 2)')
    if timeout:
        ap.add_argument('--random-timeout', type=int, default=None, metavar='T',
                        help='random: ticks after which an episode times out (default 3 ceil(S sqrt(2) / (v_max dt)), '
                             '%d for the default square)' % random_max_ticks(RANDOM_DEFAULTS['side']))


def check_random_arguments(ap, args, random_component=False):
    """ap.error when a --random-* flag is given without --scenario random.  `random_component`: a trainer's --mix
    holds a random component, which counts like --scenario random."""
    flags = RANDOM_FLAGS + (('--random-timeout',) if hasattr(args, 'random_timeout') else ())
    given = [getattr(args, f[2:].replace('-', '_')) for f in flags]
    if args.scenario != 'random' and not random_component and any(a is not None for a in given):
        if getattr(args, 'mix', None) is not None:
            ap.error('%s apply to --scenario random or a random component of --mix only' % ' / '.join(flags))
        ap.error('%s apply to --scenario random only' % ' / '.join(flags))


def random_scenario_from_arguments(ap, args):
    """The random Scenario the --random-* flags describe; ap.error for values make_scenario rejects and for a
    --random-timeout below 1.  With --random-timeout defined (a trainer) and not given, the timeout is
    random_max_ticks(side); without it (evaluate.py) the scenario keeps make_scenario's default."""
    timeout = getattr(args, 'random_timeout', None)
    if timeout is not None and timeout < 1:
        ap.error('--random-timeout must be >= 1, got %d' % timeout)
    try:
        sc = make_scenario('random', robots_per_world=args.random_robots, side=args.random_side,
                           separation=args.random_separation, min_travel=args.random_min_travel, timeout=timeout)
    except ValueError as e:
        ap.error(str(e))
    if hasattr(args, 'random_timeout') and timeout is None:
        sc = dataclasses.replace(sc, timeout=random_max_ticks(sc.layout.side))
    return sc


ARENA_FLAGS = ('--arena-robots', '--arena-count', '--arena-side', '--arena-obstacles', '--arena-seed',
               '--arena-separation', '--arena-min-travel')


def add_arena_arguments(ap, timeout=False):
    """The --arena-* flags of an arena scenario on an argparse parser; `timeout` adds --arena-timeout (training)."""
    from .arenas import ARENA_DEFAULTS as A
    ap.add_argument('--arena-robots', type=int, default=None, metavar='K',
                    help='arena: robots per world, 2..64 (default %d)' % RANDOM_DEFAULTS['robots_per_world'])
    ap.add_argument('--arena-count', type=int, default=None, metavar='T',
                    help='arena: arenas on the generated map (default %d)' % A['count'])
    ap.add_argument('--arena-side', type=float, default=None, metavar='S',
                    help='arena: side of an arena\'s interior, m (default %g)' % A['side'])
    ap.add_argument('--arena-obstacles', default=None, metavar='LO,HI',
                    help='arena: obstacles per arena, uniform in LO..HI (default %d,%d)' % A['obstacles'])
    ap.add_argument('--arena-seed', type=int, default=None, metavar='N',
                    help='arena: seed of the generated arenas; another seed gives held-out arenas (default %d)'
                         % A['seed'])
    ap.add_argument('--arena-separation', type=float, default=None, metavar='D',
                    help='arena: least start-start and goal-goal distance, m (default %g)' % A['separation'])
    ap.add_argument('--arena-min-travel', type=float, default=None, metavar='L',
                    help='arena: least start-goal distance, m (default S / 2)')
    if timeout:
        ap.add_argument('--arena-timeout', type=int, default=None, metavar='T',
                        help='arena: ticks after which an episode times out (default 3 ceil(S sqrt(2) / (v_max dt)))')


def check_arena_arguments(ap, args, arena_component=False):
    """ap.error when an --arena-* flag is given without --scenario arena (or an arena component of a trainer's --mix),
    and when a --random-* flag is given with it."""
    flags = ARENA_FLAGS + (('--arena-timeout',) if hasattr(args, 'arena_timeout') else ())
    given = lambda fl: [f for f in fl if getattr(args, f[2:].replace('-', '_'), None) is not None]
    arena = args.scenario == 'arena' or arena_component
    if not arena and given(flags):
        if getattr(args, 'mix', None) is not None:
            ap.error('%s apply to --scenario arena or an arena component of --mix only' % ' / '.join(flags))
        ap.error('%s apply to --scenario arena only' % ' / '.join(flags))
    rnd = RANDOM_FLAGS + (('--random-timeout',) if hasattr(args, 'random_timeout') else ())
    if args.scenario == 'arena' and given(rnd):
        ap.error('%s: not with --scenario arena, whose layouts the --arena-* flags shape' % ' / '.join(given(rnd)))


def arena_scenario_from_arguments(ap, args, pick):
    """The arena Scenario the --arena-* flags describe, with `pick` (0 evaluation, 1 training); ap.error for values
    make_scenario rejects and for an --arena-timeout below 1.  With --arena-timeout defined (a trainer) and not given,
    the timeout is random_max_ticks(side)."""
    timeout = getattr(args, 'arena_timeout', None)
    if timeout is not None and timeout < 1:
        ap.error('--arena-timeout must be >= 1, got %d' % timeout)
    obstacles = None
    if args.arena_obstacles is not None:
        try:
            lo, hi = (int(v) for v in args.arena_obstacles.split(','))
        except ValueError:
            ap.error('--arena-obstacles must be LO,HI (two integers), got %r' % args.arena_obstacles)
        obstacles = (lo, hi)
    try:
        sc = make_scenario('arena', robots_per_world=args.arena_robots, arenas=args.arena_count,
                           arena_side=args.arena_side, obstacles=obstacles, arena_seed=args.arena_seed,
                           separation=args.arena_separation, min_travel=args.arena_min_travel, pick=pick,
                           timeout=timeout)
    except ValueError as e:
        ap.error(str(e))
    if hasattr(args, 'arena_timeout') and timeout is None:
        sc = dataclasses.replace(sc, timeout=random_max_ticks(sc.layout.side))
    return sc


def _arena_scenario(robots_per_world, arenas, arena_side, obstacles, arena_seed, separation, min_travel, pick,
                    timeout) -> Scenario:
    from .arenas import ARENA_DEFAULTS as A, generate_arenas
    K = RANDOM_DEFAULTS['robots_per_world'] if robots_per_world is None else robots_per_world
    if not (int(K) == K and 2 <= K <= 64):
        raise ValueError(f'arena: robots_per_world must be in 2..64, got {robots_per_world}')
    K = int(K)
    S = float(np.float32(A['side'] if arena_side is None else arena_side))
    if not (math.isfinite(S) and S >= 2.0):
        raise ValueError(f'arena: side must be finite and >= 2 m, got {arena_side}')
    D = float(np.float32(A['separation'] if separation is None else separation))
    L = float(np.float32(0.5 * S if min_travel is None else min_travel))
    if not 0 <= L <= S * math.sqrt(2.0):
        raise ValueError(f'arena: min_travel must be in [0, side * sqrt(2)] = [0, {S * math.sqrt(2.0):.4g}], '
                         f'got {min_travel}')
    from .arenas import RESOLUTION
    _check_separation('arena', RESOLUTION, D, separation)
    if pick not in (0, 1):
        raise ValueError(f'arena: pick must be 0 (world) or 1 (draw), got {pick}')
    if timeout is not None and not (int(timeout) == timeout and 1 <= timeout < 2 ** 31):
        raise ValueError(f'arena: timeout must be an integer >= 1, got {timeout}')
    T = A['count'] if arenas is None else arenas
    ob = tuple(A['obstacles'] if obstacles is None else obstacles)
    seed = A['seed'] if arena_seed is None else int(arena_seed)
    m, tables = generate_arenas(T, S, ob, seed, K, D)
    zero = np.zeros((K, 4), np.float32)
    lay = ArenaLayout(D, L, int(pick), tables, int(T), S, ob, seed)
    return Scenario('arena', 2, K, 10000 if timeout is None else int(timeout), 0.7, 1, m, zero, zero.copy(), layout=lay)


def make_scenario(name: str, map_: WorldMap | None = None, robots_per_world: int | None = None,
                  radius: float | None = None, *, side: float | None = None, separation: float | None = None,
                  min_travel: float | None = None, timeout: int | None = None, arenas: int | None = None,
                  arena_side: float | None = None, obstacles: tuple | None = None, arena_seed: int | None = None,
                  pick: int = 0) -> Scenario:
    """`robots_per_world` and `radius` shape the circle scenario (see circle_layout); both None, or 50 robots with no
    radius, keep the shipped 50-row table of the reference's circle.world.

    'random' (DESIGN.md §9i): `robots_per_world` robots (default 8) on circle.world's map with the circle's tick
    constants, whose starts and goals every world draws itself (StageWorld.random_layout) in a `side` m square (default
    10), starts and goals at least `separation` m apart (default 1), each goal at least `min_travel` m from its start
    (default side / 2).  `timeout` is the tick budget of an episode (default 10000, the circle's; a training run
    passes random_max_ticks(side)).  The tables are zero; ValueError for parameters rlca_layout_random rejects or a
    square that leaves the map's free cells.

    'arena' (DESIGN.md §9v): `robots_per_world` robots (default 8) per world in one of `arenas` walled arenas (default
    64) of `arena_side` m (default 10) with U{lo..hi} = `obstacles` (default 4..10) random obstacles each, generated from
    `arena_seed` (default 0; arenas.generate_arenas), on that map with the circle's tick constants.  Starts and goals
    lie in the arena's placeable cells, `separation` (default 1.2: at 0.2 m rlca_layout_random's bound
    2 (r_c + sqrt(2) res) is 1.147 m) and `min_travel` (default arena_side / 2) as for random; `pick` 0 puts world w in arena (world_offset + w) mod T (evaluation), 1 draws an arena at every layout
    (training).  `timeout` as for random.  ValueError for parameters rlca_layout_arena rejects and for arenas the
    generator refuses, a map off the small-map path included."""
    name = name.lower()
    arena_args = (arenas, arena_side, obstacles, arena_seed)
    if name not in ('random', 'arena') and (side is not None or separation is not None or min_travel is not None or
                                            timeout is not None):
        raise ValueError('side, separation, min_travel and timeout shape the random scenario only (and, but for side, '
                         'the arena scenario)')
    if name != 'arena' and (any(a is not None for a in arena_args) or pick != 0):
        raise ValueError('arenas, arena_side, obstacles, arena_seed and pick shape the arena scenario only')
    if name == 'arena':
        if radius is not None or side is not None or map_ is not None:
            raise ValueError('radius, side and map_ do not shape the arena scenario: it generates its map')
        return _arena_scenario(robots_per_world, *arena_args, separation, min_travel, pick, timeout)
    if name == 'random':
        if radius is not None:
            raise ValueError('radius shapes the circle scenario only')
        m = map_ or load_map(os.path.join(ASSETS, 'circle_map.npz'))
        K = RANDOM_DEFAULTS['robots_per_world'] if robots_per_world is None else robots_per_world
        S = RANDOM_DEFAULTS['side'] if side is None else side
        D = RANDOM_DEFAULTS['separation'] if separation is None else separation
        lay = random_layout_params(m, K, S, D, 0.5 * float(S) if min_travel is None else min_travel)
        K = int(K)
        zero = np.zeros((K, 4), np.float32)
        if timeout is not None and not (int(timeout) == timeout and 1 <= timeout < 2 ** 31):
            raise ValueError(f'random: timeout must be an integer >= 1, got {timeout}')
        T = 10000 if timeout is None else int(timeout)
        return Scenario('random', 2, K, T, 0.7, 1, m, zero, zero.copy(), layout=lay)
    if name == 'stage1':
        m = map_ or load_map(os.path.join(ASSETS, 'stage1_map.npz'))
        R = robots_per_world or 24
        init = np.zeros((R, 4), np.float32)
        k = min(R, len(m.init_poses))
        init[:k, :3] = m.init_poses[:k]
        goal = np.zeros((R, 4), np.float32)
        return Scenario('stage1', 0, R, 150, 1.05, 0, m, init, goal)
    if name == 'stage2':
        m = map_ or load_map(os.path.join(ASSETS, 'stage2_map.npz'))
        t = _tables()['stage2']
        R = 44
        init = np.zeros((R, 4), np.float32)
        init[:, :3] = np.asarray(t['init_pose'], np.float64)
        goal = np.zeros((R, 4), np.float32)
        g = np.asarray(t['goal_point'], np.float64)          # 34 rows (model/utils.py:55-63)
        goal[:len(g), :2] = g
        init[34:44, 3] = 1.0                                  # stage_world2.py:211 random spawn
        goal[34:44, 2] = 1.0                                  # stage_world2.py:165 random goal
        grp = t['groups']                                     # model/utils.py:83 group boundaries
        for gi, (a, b) in enumerate(zip(grp[:-1], grp[1:])):
            goal[a:b, 3] = gi
        return Scenario('stage2', 1, R, 200, 1.05, 1, m, init, goal, groups=tuple(t['groups']))
    if name == 'circle':
        m = map_ or load_map(os.path.join(ASSETS, 'circle_map.npz'))
        if radius is None and robots_per_world in (None, 50):
            t = _tables()['circle']
            R = 50
            init = np.zeros((R, 4), np.float32)
            init[:, :3] = np.asarray(t['init_pose'], np.float64)
            goal = np.zeros((R, 4), np.float32)
            goal[:, :2] = np.asarray(t['goal_point'], np.float64)
        else:
            init, goal = circle_layout(m, 50 if robots_per_world is None else robots_per_world,
                                       25.0 if radius is None else radius)
            R = len(init)
        return Scenario('circle', 2, R, 10000, 0.7, 1, m, init, goal)
    raise ValueError(f'unknown scenario {name!r}')


def fill_config(cfg, sc: Scenario, *, num_worlds: int, beams: int, raw_beams: int | None = None,
                auto_reset: bool = False, seed: int = 0, world_offset: int = 0, max_reject: int = 4096):
    """Fill a ctypes config structure (EnvConfig or the oracle's mirror) from a Scenario."""
    import ctypes as C
    f32 = lambda v: C.c_float(v).value
    m = sc.map
    cfg.robots_per_world = sc.robots_per_world
    cfg.num_worlds = num_worlds
    cfg.beams = beams
    cfg.raw_beams = raw_beams if raw_beams is not None else max(COMMON['raw_beams'], beams)
    cfg.grid_w, cfg.grid_h = m.grid_w, m.grid_h
    cfg.origin_cx, cfg.origin_cy = m.origin_cx, m.origin_cy
    cfg.resolution = m.resolution
    cfg.ppm = f32(1.0 / m.resolution)
    cfg.dt = COMMON['dt']
    cfg.inv_dt = np.float32(1.0) / np.float32(COMMON['dt'])
    cfg.range_max = COMMON['range_max']
    cfg.range_cells = np.float32(cfg.ppm) * np.float32(COMMON['range_max'])
    cfg.fov = COMMON['fov']
    for k in ('half_len', 'half_wid', 'goal_radius', 'reward_arrive', 'reward_collision', 'progress_gain',
              'w_penalty', 'v_min', 'v_max', 'w_min', 'w_max'):
        setattr(cfg, k, COMMON[k])
    cfg.w_threshold = sc.w_threshold
    cfg.timeout = sc.timeout
    cfg.pre_distance_zero = sc.pre_distance_zero
    cfg.scenario = sc.scenario_id
    cfg.auto_reset = int(auto_reset)
    cfg.max_reject = max_reject
    cfg.world_offset = world_offset
    cfg.seed = seed
    return cfg
