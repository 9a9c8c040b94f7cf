"""Numpy restatement of the progress metrics (DESIGN.md §9o), written from the definitions, not from
csrc/rlca_progress.cu: which tick is folded into which episode, the per-episode state (closest, progress reference and
ticks since progress, still run and still ticks, rotation, robot near), the cause of a time-out or an unfinished
episode, and the float64 reduction.  float32 arithmetic, one rounding per operation."""
import numpy as np

_F = np.float32
COLUMNS = tuple(g + '_' + k for g in ('timeout', 'unfinished')
                for k in ('frozen', 'stalled', 'slow', 'robot_near', 'folded', 'sum_closest', 'sum_closest_sq')) + \
    ('sum_still_ticks', 'sum_ticks', 'reached', 'sum_rotation', 'sum_rotation_sq')
PI = _F(3.14159274101257324219)
TWO_PI = _F(6.28318548202514648438)


def wrap(a):
    """The tick's wrap: one step of 2 pi towards (-pi, pi]."""
    a = _F(a)
    if a > PI:
        return _F(a - TWO_PI)
    if a <= -PI:
        return _F(a + TWO_PI)
    return a


def cause(window, run, since, near):
    c = 1 if run >= window else 2 if since >= window else 3
    return c + (4 if near else 0)


class Episode:
    """The running state of one robot's episode; ticks == 0 means no folded tick yet."""

    def __init__(self):
        self.closest = _F(0)
        self.ref = _F(0)
        self.rotation = _F(0)
        self.near = False
        self.since = self.run = self.still = self.ticks = 0


class Tracker:
    """The episode tracker's boundaries (closed, count) and the progress fold next to them."""

    def __init__(self, cfg, episodes, window=50, progress_dist=0.1, still_dist=0.005, block_dist=1.0):
        self.R, self.E = cfg.robots_per_world, int(episodes)
        self.window = int(window)
        self.progress_dist, self.still_dist, self.block_dist = _F(progress_dist), _F(still_dist), _F(block_dist)
        N = cfg.robots_per_world * cfg.num_worlds
        self.closed = np.full(N, -1, np.int32)
        self.count = np.zeros(N, np.int32)
        self.open = np.ones(N, np.int32)
        self.ep = [Episode() for _ in range(N)]
        self.records = np.zeros((N, self.E, 4), np.float32)
        self.causes = np.zeros((N, self.E), np.uint8)
        self.results = np.zeros((N, self.E, 4), np.float32)        # the tracker's records: result code in [..., 0]

    def state(self):
        """The library's layout of the running state."""
        running = np.array([(e.closest, e.ref, e.rotation, _F(1) if e.near else _F(0)) for e in self.ep], np.float32)
        counters = np.array([(e.since, e.run, e.still, e.ticks) for e in self.ep], np.int32)
        return dict(running=running, counters=counters, records=self.records, causes=self.causes)

    def _near(self, pose_out, a):
        """Another robot of a's world, whatever its state, with its centre strictly within block_dist of a's."""
        w = a // self.R
        x, y = _F(pose_out[a][0]), _F(pose_out[a][1])
        for b in range(w * self.R, (w + 1) * self.R):
            if b == a:
                continue
            dx, dy = _F(_F(pose_out[b][0]) - x), _F(_F(pose_out[b][1]) - y)
            if np.sqrt(_F(_F(dx * dx) + _F(dy * dy))) < self.block_dist:
                return True
        return False

    def tick(self, pose_in, meta_in, pose_out, flags, meta_out=None):
        for a in range(len(pose_in)):
            done, crashed, result, respawned = (int(v) for v in flags[a])
            epi = int(meta_in[a][1])
            e = self.ep[a]
            if self.closed[a] != epi:                                 # the tick belongs to a tracked episode
                if not respawned:                                     # folded
                    d = _F(pose_out[a][3])
                    dx, dy = _F(_F(pose_out[a][0]) - _F(pose_in[a][0])), _F(_F(pose_out[a][1]) - _F(pose_in[a][1]))
                    s = np.sqrt(_F(_F(dx * dx) + _F(dy * dy)))
                    if e.ticks == 0:
                        e.closest, e.ref, e.since = d, d, 0
                    else:
                        e.closest = min(e.closest, d)
                        if d <= _F(e.ref - self.progress_dist):
                            e.ref, e.since = d, 0
                        else:
                            e.since += 1
                    if s < self.still_dist:
                        e.run += 1
                        e.still += 1
                    else:
                        e.run = 0
                    e.rotation = _F(e.rotation + abs(wrap(_F(_F(pose_out[a][2]) - _F(pose_in[a][2])))))
                    e.near = self._near(pose_out, a)
                    e.ticks += 1
                if result != 0:                                       # the episode ends: record into slot count
                    c = int(self.count[a])
                    if c < self.E:
                        self.records[a, c] = (e.closest, e.rotation, e.still, e.ticks)
                        self.causes[a, c] = cause(self.window, e.run, e.since, e.near) if result == 3 else 0
                        self.results[a, c, 0] = result
                    self.count[a] = c + 1
                    self.closed[a] = epi
                    self.ep[a] = Episode()
            if respawned:
                self.ep[a] = Episode()
            if meta_out is not None:
                self.open[a] = int(self.closed[a] != int(meta_out[a][1]))


def reduce(window, R, records, causes, running, counters, results, count, open_, mask=None, split=False, want=0,
           world=0):
    """The partials of one world, float64, agents then records; `results[..., 0]` is the tracker's result code."""
    s = dict.fromkeys(COLUMNS, 0.0)
    E = records.shape[1]

    def group(g, c, closest, folded):
        if c & 3:
            s[g + '_' + ('frozen', 'stalled', 'slow')[(c & 3) - 1]] += 1.0
        if c & 4:
            s[g + '_robot_near'] += 1.0
        if folded:
            d = float(closest)
            s[g + '_folded'] += 1.0
            s[g + '_sum_closest'] += d
            s[g + '_sum_closest_sq'] += d * d

    for r in range(R):
        a = world * R + r
        if split and (mask[a] != 0) != bool(want):
            continue
        for i in range(min(int(count[a]), E)):
            closest, rot, still, ticks = (float(v) for v in records[a, i])
            res = int(results[a, i, 0])
            s['sum_still_ticks'] += still
            s['sum_ticks'] += ticks
            if res == 3:
                group('timeout', int(causes[a, i]), closest, ticks > 0)
            if res == 1:
                s['reached'] += 1.0
                s['sum_rotation'] += rot
                s['sum_rotation_sq'] += rot * rot
        if count[a] < E and open_[a]:
            since, run, _, ticks = (int(v) for v in counters[a])
            group('unfinished', cause(window, run, since, running[a][3] != 0), running[a][0], ticks > 0)
    return np.array([s[k] for k in COLUMNS], np.float64)
