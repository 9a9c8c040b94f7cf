"""Numpy restatement of the latency rule (include/rlca.h, DESIGN.md §9q), written from the rule, not the kernel.

Delays: an agent starting an episode draws d = lo + floor((hi - lo + 1) w0 / 2^32), w0 the first Philox-4x32-10 word
(layout_ref.philox) of (global agent, draw, 0, purpose | stream << 8) under the key (seed lo, seed hi), global agent =
(world_offset + w) R + r, purposes 0xE4 (scan) and 0xE5 (command).

Instead of rings, each agent keeps the list of its episode's true frames and issued commands:
- scan: a fresh row's list restarts at its newest frame and its stack is left alone; any other row appends its newest
  frame and reads frames[-1 - d], or the episode's first frame while the list is no longer than d;
- command: a fresh row's list restarts empty; every row appends the issued command and executes commands[-1 - l], or
  the episode's first command while the list is no longer than l.
A range whose hi is 0 leaves everything as it is."""
import numpy as np

from layout_ref import philox

PURPOSE_SCAN, PURPOSE_CMD = 0xE4, 0xE5
_M32 = 0xFFFFFFFF


def delays(seed, agents, draw, lo, hi, purpose, stream=0):
    """int64 delays of the global agents `agents` drawn at call `draw`"""
    a = np.asarray(agents, np.uint64)
    full = lambda v: np.full(a.shape, v, np.uint64)
    w0 = philox((a, full(draw), full(0), full(purpose | (stream << 8))), int(seed) & _M32, int(seed) >> 32)[0]
    return lo + ((np.uint64(hi - lo + 1) * w0) >> np.uint64(32)).astype(np.int64)


class Latency:
    """The rule for N = R W agents of one env handle; `scan` and `action` keep their own call counters."""

    def __init__(self, R, W, scan_delay, command_delay, seed, world_offset=0, stream=0):
        self.N = R * W
        self.agents = np.uint64(world_offset * R) + np.arange(self.N, dtype=np.uint64)
        self.sr, self.cr, self.seed, self.stream = tuple(scan_delay), tuple(command_delay), seed, stream
        self.scan_calls = self.action_calls = 0
        self.d = np.zeros(self.N, np.int64)
        self.l = np.zeros(self.N, np.int64)
        self.frames = [[] for _ in range(self.N)]
        self.cmds = [[] for _ in range(self.N)]

    def scan(self, stack, flags=None):
        """in place on the (N, 3, B) float32 stack"""
        t = self.scan_calls
        self.scan_calls += 1
        if self.sr[1] == 0:
            return stack
        fresh = np.ones(self.N, bool) if flags is None else np.asarray(flags)[:, 3] != 0
        drawn = delays(self.seed, self.agents, t, self.sr[0], self.sr[1], PURPOSE_SCAN, self.stream)
        for a in range(self.N):
            newest = stack[a, 2].copy()
            if fresh[a]:
                self.frames[a] = [newest]
                self.d[a] = drawn[a]
                continue
            f = self.frames[a]
            f.append(newest)
            del f[1:max(1, len(f) - 9)]           # the first frame and the last 9 are all a delay can reach
            stack[a, 2] = f[-1 - self.d[a]] if len(f) > self.d[a] else f[0]
        return stack

    def action(self, cmd, flags=None):
        """the executed (N, 2) float32 command for the issued command `cmd`"""
        t = self.action_calls
        self.action_calls += 1
        cmd = np.asarray(cmd, np.float32)
        if self.cr[1] == 0:
            return cmd.copy()
        fresh = np.ones(self.N, bool) if flags is None else np.asarray(flags)[:, 3] != 0
        drawn = delays(self.seed, self.agents, t, self.cr[0], self.cr[1], PURPOSE_CMD, self.stream)
        out = np.zeros((self.N, 2), np.float32)
        for a in range(self.N):
            if fresh[a]:
                self.cmds[a] = []
                self.l[a] = drawn[a]
            q = self.cmds[a]
            q.append(cmd[a].copy())
            del q[1:max(1, len(q) - 9)]
            out[a] = q[-1 - self.l[a]] if len(q) > self.l[a] else q[0]
        return out
