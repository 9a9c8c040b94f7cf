"""Training on a mix of scenarios (DESIGN.md §9l): several env handles, one per scenario, side by side in one rollout.

Component k of a mix owns the contiguous agent columns [a_k, b_k) of the trainer's Rollout, in the order the components
were given; every tick runs one policy forward over all columns and one env tick per component on its slices, and
every PPO update trains on all columns together.  This module holds the host-side plan (names, world counts, column
ranges, per-rank world offsets) and the alignment check of the rollout slices; trainer.run composes the handles.
"""
from __future__ import annotations

from dataclasses import dataclass

# The scenarios a mix may hold, and the auto_reset each trains with: stage 2 and the circle re-spawn a group inside the
# tick (auto_reset 2, as ppo_stage2.py trains them alone); a random scenario re-lays finished worlds between ticks
# (auto_reset 0 with env.live and relayout_finished, §9k), and so does an arena scenario (§9v).  Stage 1 re-spawns per robot and trains with stage 1's
# update, so it cannot share a stage-2 update.
MIX_SCENARIOS = ('stage2', 'circle', 'random', 'arena')
MIX_AUTO_RESET = {'stage2': 2, 'circle': 2, 'random': 0, 'arena': 0}

# Byte alignment of a component's slice of each rollout buffer: the element type rlca_env_step reads or writes a row
# with (action float2, reward float, flags uchar4, gs and eplog float4), and 16 bytes for the scan FIFO, which
# rlca_stack_refresh requires and the tick's 4-beams-per-lane lidar path needs.
SLICE_ALIGN = {'action': 8, 'reward': 4, 'flags': 4, 'gs': 16, 'eplog': 16, 'stack': 16}


@dataclass(frozen=True)
class Component:
    name: str                  # 'stage2', 'circle', 'random' or 'arena'
    worlds: int                # worlds of this component on one GPU
    robots_per_world: int
    world_offset: int          # global index of this rank's first world of the component
    cols: tuple                # [a, b): the component's agent columns of the rollout

    @property
    def n(self):
        return self.worlds * self.robots_per_world


def parse_mix(text):
    """[(name, worlds), ...] of a --mix value such as 'stage2:31,random:128,circle:14', in the order given.
    ValueError for a malformed entry, stage 1, an unknown or repeated name, or a world count below 1."""
    out = []
    for item in text.split(','):
        name, sep, count = item.strip().partition(':')
        name = name.strip().lower()
        if not sep or not name:
            raise ValueError(f'--mix entries are name:worlds, got {item!r}')
        try:
            w = int(count)
        except ValueError:
            raise ValueError(f'--mix: the world count of {name} must be an integer, got {count!r}') from None
        if name == 'stage1':
            raise ValueError('--mix: stage 1 cannot be mixed (it re-spawns each robot on its own and trains with stage '
                             "1's update)")
        if name not in MIX_SCENARIOS:
            raise ValueError(f'--mix: unknown scenario {name!r} (one of {", ".join(MIX_SCENARIOS)})')
        if any(n == name for n, _ in out):
            raise ValueError(f'--mix: {name} appears more than once')
        if w < 1:
            raise ValueError(f'--mix: {name} needs at least 1 world, got {w}')
        out.append((name, w))
    return out


def plan(mix, robots_per_world, rank=0):
    """The Components of a parsed mix on GPU `rank`: robots_per_world maps each name to its robots per world.  Rank r
    gets world_offset r * W_k in component k, so every component shards exactly as a single-scenario run of that
    scenario with W_k worlds per GPU; columns follow the order of `mix`."""
    comps, a = [], 0
    for name, w in mix:
        r = int(robots_per_world[name])
        comps.append(Component(name, int(w), r, int(rank) * int(w), (a, a + int(w) * r)))
        a += int(w) * r
    return comps


def check_aligned(name, view, align):
    """ValueError unless every row of `view` (a component's column slice of a rollout buffer, for every tick) starts
    on an `align`-byte boundary: its start and the byte step of every axis but the last must be multiples of
    `align`.  `name` is the buffer's name in the message."""
    off = view.data_ptr() % align
    steps = [s * view.element_size() for s in view.stride()[:-1]]
    if off or any(s % align for s in steps):
        raise ValueError(f'rollout slice {name} is not {align}-byte aligned (start offset {off} bytes, steps {steps} '
                         f'bytes): the kernels read its rows {align} bytes at a time')
