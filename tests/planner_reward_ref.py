"""A float64 restatement of the planner's geodesic progress shaping (DESIGN.md §9x) for the CPU tests: the potential
excess psi of a row from tests/planner_ref.py's waypoint, the shaped reward of a tick and the shaped return of an
episode."""
import math

import planner_ref as ref


def psi(label, ocx, ocy, ppm, res, D, rect, entry_ok, pose, goal):
    """(status, psi) of one row in float64: 0 unless the row steers by a waypoint w (status 1), else the distance to w
    plus D(w's cell) res / 70, less the straight-line distance pose[3] the tick stored."""
    s, wp, ch, k = ref.waypoint(label, ocx, ocy, ppm, res, D, rect, entry_ok, pose, goal)
    if s != 1:
        return s, 0.0
    x, y = ch[k]
    L = ref.field_at(D, rect, x, y) * res / 70.0
    return s, math.hypot(wp[0] - float(pose[0]), wp[1] - float(pose[1])) + L - float(pose[3])


def shaped_reward(reward, flags, psi_prev, psi_now, gain):
    """The tick's reward plus gain (psi_prev - psi) on a non-terminal tick (flags[0] == 0); else the tick's."""
    return float(reward) + (float(gain) * (float(psi_prev) - float(psi_now)) if flags[0] == 0 else 0.0)


def shaped_return(tick_rewards, flags, psis, gain):
    """Sum of an episode's shaped rewards: tick_rewards[i] and flags[i] of its ticks, psis[0] at its start and psis[i + 1]
    after tick i."""
    return sum(shaped_reward(r, f, psis[i], psis[i + 1], gain) for i, (r, f) in enumerate(zip(tick_rewards, flags)))
