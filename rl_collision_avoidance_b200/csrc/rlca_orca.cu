// rlca_orca.cu — ORCA-DD baseline controller on the device (sm_90a), C ABI in include/rlca.h, DESIGN.md §9d.
//
// Reciprocal collision avoidance (van den Berg, Guy, Lin, Manocha, "Reciprocal n-body collision avoidance", 2011,
// §4-5) for every robot of every world, from the simulator state the next rlca_env_step reads, followed by a
// differential-drive heading tracker that turns the ORCA velocity into a raw (v, w) action.  This is not NH-ORCA: no
// tracking-error radius, no non-holonomic constraint set, no static obstacles.
//
// One warp per agent, 8 agents per CTA.  The lanes build the half-planes of the world's other robots in parallel and
// compact the in-range ones into per-warp shared memory in robot-index order.  The 2-D LP is the incremental one; the
// 1-D LP of line i scans lines 0..i-1 across the lanes and combines the bounds with warp max / min (exact) and a ballot,
// so it equals the serial loop bit for bit.  The least-penetration fallback (3-D LP) builds its projected lines the same
// way.  rlca_orca_action_host runs the serial loops over the same per-line functions; -fmad=false on the device and
// -ffp-contract=off on the host make both round alike.
//
// NH-ORCA (Alonso-Mora, Breitenmoser, Rufli, Beardsley, Siegwart, "Optimal reciprocal collision avoidance for multiple
// non-holonomic robots", DARS 2010; DESIGN.md §9e) is the same kernel with three changes: every radius grows by the
// tracking error E, the edges of a convex polygon P inside the velocities the robot can track within E come first in the
// LP as hard lines (one per lane, rotated by the heading), and the action is the arc that tracks the chosen velocity.
// P is built on the host in float64 (nh_build_polygon).
//
// Static obstacles (DESIGN.md §9f), for both controllers: the boundary of the occupied cells of the static grid as
// closed loops of segments (built once on the host, orca_obstacles_build), a per-bin candidate list, and RVO2's
// obstacle half-planes (van den Berg et al. 2011, §6) with horizon tau_o and full responsibility, placed after P's edges
// and before the agent lines and kept hard in the least-penetration fallback.
//
// The non-cooperative driver (DESIGN.md §9h) overwrites the actions of masked agents with ORCA-DD's answer for an agent
// without neighbours: straight to the goal, ignoring everyone else.
//
// The hybrid controller (DESIGN.md §9j) switches each agent's policy action by the nearest return of its newest scan:
// the §9h driver in free space, the policy's action with a capped speed near obstacles, the policy's action otherwise.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include <string.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define ORCA_THREADS 256
#define ORCA_WARPS (ORCA_THREADS / 32)
#define ORCA_MAX_LINES (RLCA_MAX_ROBOTS_PER_WORLD - 1)
#define NH_ORCA_VERTS RLCA_NH_ORCA_VERTS
#define NH_MAX_LINES (NH_ORCA_VERTS + ORCA_MAX_LINES)
#define OBS_CAND RLCA_ORCA_MAP_MAX_CANDIDATES
#define OBS_LINES RLCA_ORCA_MAP_MAX_LINES
#define ALL_MAX_LINES (NH_ORCA_VERTS + OBS_LINES + ORCA_MAX_LINES)
#define OBS_BIN ((double)RLCA_ORCA_MAP_BIN)     // side of a lookup bin, m
#define OBS_SLACK 1e-3              // a bin's list holds the segments within max_range + this of the bin, m
#define ORCA_PARALLEL_EPS 1e-5f     // |det| of two unit directions below which lines count as parallel
#define ORCA_STILL 1e-6f            // ORCA speeds at or below this give the action (0, 0)
#define FULL_MASK 0xffffffffu

// Half-plane {v : det(d, v - p) >= 0}: the allowed side is left of the unit direction d.
struct OrcaLine {
    float px, py, dx, dy;
};

struct OrcaAgent {
    float px, py, vx, vy, ct, st;
};

struct OrcaParams {
    float r;            // combined radius 2 * radius
    float nd2;          // neighbour_dist^2
    float inv_tau, inv_dt;
    float v_max, w_min, w_max, gain;
};

// NH-ORCA's polygon P and tracker parameters.
struct NhParams {
    int nv;                         // vertices of P = its hard lines
    float heading_time, v_min;
    OrcaLine edge[NH_ORCA_VERTS];   // in the robot frame: vertex k, unit direction to vertex k + 1 (P on the left)
};

// One boundary segment of the static map, occupied cells on its left: start vertex (x0, y0), end vertex (x1, y1), unit
// direction, the directions of the previous and next segments of its loop, and the convex flags of both vertices.
struct ObsSeg {
    float x0, y0, x1, y1;
    float dx, dy, pdx, pdy;
    float ndx, ndy;
    int32_t convex0, convex1;
    int32_t prev, next;
    int32_t pad[2];
};

// The obstacle set as one launch reads it (device or host pointers) and the per-call parameters.
struct ObsParams {
    const ObsSeg *seg;
    const int32_t *bin_off;         // nbx * nby + 1 offsets into bin_idx
    const int32_t *bin_idx;         // per bin: the segments within max_range of it, in index order
    float bx0, by0, inv_bin;        // world position of bin (0, 0)'s corner, 1 / bin side
    int32_t nbx, nby;
    float range2;                   // (tau_o v_max + r_o)^2
    float inv_tau, r, rt;           // 1 / tau_o, r_o, r_o / tau_o
};

__host__ __device__ __forceinline__ float det2(float ax, float ay, float bx, float by) { return ax * by - ay * bx; }

// Position, heading and current velocity of agent a: the last clipped command goal.z along the heading, 0 when the
// last move was reverted (stall flag meta.z).
__host__ __device__ __forceinline__ OrcaAgent orca_agent(const float4 *pose, const float4 *goal, const int4 *meta, int a)
{
    const float4 p = pose[a];
    float s, c;
    dev_sincosf(p.z, s, c);
    const float v = meta[a].z ? 0.0f : goal[a].z;
    OrcaAgent g;
    g.px = p.x; g.py = p.y; g.vx = v * c; g.vy = v * s; g.ct = c; g.st = s;
    return g;
}

__host__ __device__ __forceinline__ bool orca_in_range(const OrcaAgent &a, const OrcaAgent &b, float nd2)
{
    const float dx = b.px - a.px, dy = b.py - a.py;
    return dx * dx + dy * dy < nd2;
}

// The ORCA half-plane agent a gets from neighbour b: u is the smallest change of the relative velocity that takes it
// to the boundary of the velocity obstacle (truncated cone with horizon tau; when the pair already overlaps, the disk of
// one time step), and a takes half of it.  False when the relative velocity is exactly the centre of the one-step disk,
// where no direction is preferred; the neighbour then adds no line.
__host__ __device__ __forceinline__ bool orca_line(const OrcaAgent &a, const OrcaAgent &b, const OrcaParams &q,
                                                   OrcaLine &l)
{
    const float rpx = b.px - a.px, rpy = b.py - a.py;
    const float rvx = a.vx - b.vx, rvy = a.vy - b.vy;
    const float dist2 = rpx * rpx + rpy * rpy, r = q.r, r2 = r * r;
    float ux, uy, dx, dy;
    if (dist2 > r2) {
        const float wx = rvx - q.inv_tau * rpx, wy = rvy - q.inv_tau * rpy;    // cut-off centre -> relative velocity
        const float w2 = wx * wx + wy * wy, dot1 = wx * rpx + wy * rpy;
        if (dot1 < 0.0f && dot1 * dot1 > r2 * w2) {
            // nearest boundary point on the cut-off arc
            const float wl = sqrtf(w2), nx = wx / wl, ny = wy / wl;
            dx = ny; dy = -nx;
            const float k = r * q.inv_tau - wl;
            ux = k * nx; uy = k * ny;
        } else {
            // nearest boundary point on a leg: the direction is the leg's, pointing away from the apex on the left
            // leg and towards it on the right one, so that the cone is on the right
            const float leg = sqrtf(dist2 - r2);
            if (det2(rpx, rpy, wx, wy) > 0.0f) {
                dx = (rpx * leg - rpy * r) / dist2;
                dy = (rpx * r + rpy * leg) / dist2;
            } else {
                dx = -(rpx * leg + rpy * r) / dist2;
                dy = -(rpy * leg - rpx * r) / dist2;
            }
            const float t = rvx * dx + rvy * dy;
            ux = t * dx - rvx; uy = t * dy - rvy;
        }
    } else {
        const float wx = rvx - q.inv_dt * rpx, wy = rvy - q.inv_dt * rpy;
        const float wl = sqrtf(wx * wx + wy * wy);
        if (!(wl > 0.0f)) return false;
        const float nx = wx / wl, ny = wy / wl;
        dx = ny; dy = -nx;
        const float k = r * q.inv_dt - wl;
        ux = k * nx; uy = k * ny;
    }
    l.px = a.vx + 0.5f * ux;
    l.py = a.vy + 0.5f * uy;
    l.dx = dx;
    l.dy = dy;
    return true;
}

// v_pref = d * min(v_max / |d|, 1 / dt) with d = goal - p; 0 on the goal.
__host__ __device__ __forceinline__ void orca_pref(const OrcaAgent &a, float4 goal, const OrcaParams &q, float &ox,
                                                   float &oy)
{
    const float dx = goal.x - a.px, dy = goal.y - a.py, d = sqrtf(dx * dx + dy * dy);
    if (d > 0.0f) {
        const float k = fminf(q.v_max / d, q.inv_dt);
        ox = dx * k; oy = dy * k;
    } else {
        ox = 0.0f; oy = 0.0f;
    }
}

// Start of the 2-D LP: the optimum on the speed disk alone.
__host__ __device__ __forceinline__ void lp2_start(float radius, float ox, float oy, bool dir_opt, float &rx, float &ry)
{
    if (dir_opt) {
        rx = ox * radius; ry = oy * radius;
    } else if (ox * ox + oy * oy > radius * radius) {
        const float n = sqrtf(ox * ox + oy * oy);
        rx = ox / n * radius; ry = oy / n * radius;
    } else {
        rx = ox; ry = oy;
    }
}

__host__ __device__ __forceinline__ bool violates(const OrcaLine &l, float rx, float ry)
{
    return det2(l.dx, l.dy, l.px - rx, l.py - ry) > 0.0f;
}

// 1-D LP on line i: the interval [tl, tr] of p + t d inside the speed disk; false when the line misses the disk.
__host__ __device__ __forceinline__ bool lp1_range(const OrcaLine &l, float radius, float &tl, float &tr)
{
    const float dot = l.px * l.dx + l.py * l.dy;
    const float disc = dot * dot + radius * radius - (l.px * l.px + l.py * l.py);
    if (disc < 0.0f) return false;
    const float s = sqrtf(disc);
    tl = -dot - s;
    tr = -dot + s;
    return true;
}

// The bound line k puts on t along line i: 1 = t <= b, -1 = t >= b, 0 = none (parallel, i inside k),
// 2 = infeasible (parallel, i outside k).
__host__ __device__ __forceinline__ int lp1_bound(const OrcaLine &li, const OrcaLine &lk, float &b)
{
    const float den = det2(li.dx, li.dy, lk.dx, lk.dy);
    const float num = det2(lk.dx, lk.dy, li.px - lk.px, li.py - lk.py);
    if (fabsf(den) <= ORCA_PARALLEL_EPS) return num < 0.0f ? 2 : 0;
    b = num / den;
    return den >= 0.0f ? 1 : -1;
}

// The optimum on line i within [tl, tr]: nearest to opt, or furthest along the direction opt.
__host__ __device__ __forceinline__ void lp1_pick(const OrcaLine &l, float tl, float tr, float ox, float oy,
                                                  bool dir_opt, float &rx, float &ry)
{
    float t;
    if (dir_opt) t = (ox * l.dx + oy * l.dy > 0.0f) ? tr : tl;
    else t = fminf(fmaxf(l.dx * (ox - l.px) + l.dy * (oy - l.py), tl), tr);
    rx = l.px + t * l.dx;
    ry = l.py + t * l.dy;
}

// Line of the least-penetration program of line i for an earlier line j: the points v where the penetrations into i and
// j are equal, det(e, v - p_i) = det(d_j, p_j - p_i) with e = d_j - d_i.  Its point is the one nearest to p_i, not the
// crossing of i and j: for nearly parallel i and j the crossing lies far away (1e4 m for lines 0.1 m apart at
// |det(d_i, d_j)| = 1e-5), and rounding it moves the line by up to 1e-3 m across i, which can cut the optimum off and
// leave the fallback stuck above it.  False when j is parallel to i and points the same way (it never binds before i
// does).
__host__ __device__ __forceinline__ bool lp3_line(const OrcaLine &li, const OrcaLine &lj, OrcaLine &o)
{
    if (fabsf(det2(li.dx, li.dy, lj.dx, lj.dy)) <= ORCA_PARALLEL_EPS && li.dx * lj.dx + li.dy * lj.dy > 0.0f)
        return false;
    const float h = det2(lj.dx, lj.dy, lj.px - li.px, lj.py - li.py);
    const float ex = lj.dx - li.dx, ey = lj.dy - li.dy, e2 = ex * ex + ey * ey, el = sqrtf(e2), k = h / e2;
    o.px = li.px - k * ey;
    o.py = li.py + k * ex;
    o.dx = ex / el;
    o.dy = ey / el;
    return true;
}

// Heading tracker: the ORCA velocity in the robot's frame (c along the heading, s to its left) -> raw (v, w).
__host__ __device__ __forceinline__ float2 orca_track(const OrcaAgent &a, float vx, float vy, const OrcaParams &q)
{
    const float n = sqrtf(vx * vx + vy * vy);
    if (n <= ORCA_STILL) return make_float2(0.0f, 0.0f);
    const float c = vx * a.ct + vy * a.st, s = vy * a.ct - vx * a.st;
    if (c > 0.0f) return make_float2(fminf(c, q.v_max), fminf(fmaxf(q.gain * s / n, q.w_min), q.w_max));
    return make_float2(0.0f, s >= 0.0f ? q.w_max : q.w_min);
}

// Edge e of P (robot frame) rotated by agent a's heading into the world frame.
__host__ __device__ __forceinline__ OrcaLine nh_hard_line(const OrcaAgent &a, const OrcaLine &e)
{
    OrcaLine l;
    l.px = a.ct * e.px - a.st * e.py;
    l.py = a.st * e.px + a.ct * e.py;
    l.dx = a.ct * e.dx - a.st * e.dy;
    l.dy = a.st * e.dx + a.ct * e.dy;
    return l;
}

// Arc tracker: the velocity at angle th from the heading, speed V, -> turn at w = th / T_th for T_th =
// max(T, th / w_max) (th < 0: w_min) while driving at v* = V (th/2) cot(th/2), then straight at V.
__host__ __device__ __forceinline__ float2 nh_track(const OrcaAgent &a, float vx, float vy, const OrcaParams &q,
                                                    const NhParams &h)
{
    const float n = sqrtf(vx * vx + vy * vy);
    if (n <= ORCA_STILL) return make_float2(0.0f, 0.0f);
    const float c = vx * a.ct + vy * a.st, s = vy * a.ct - vx * a.st;
    const float th = dev_atan2f(s, c);
    const float turn = fmaxf(h.heading_time, th / (th >= 0.0f ? q.w_max : q.w_min));
    const float half = 0.5f * th;
    float v = n;
    if (half != 0.0f) {
        float sh, ch;
        dev_sincosf(half, sh, ch);
        v = n * (half * ch / sh);
    }
    return make_float2(fminf(fmaxf(v, h.v_min), q.v_max), fminf(fmaxf(th / turn, q.w_min), q.w_max));
}

// ------------------------------------------------------------------------------------ static obstacles (§9f)
__host__ __device__ __forceinline__ uint32_t float_bits(float x)
{
#ifdef __CUDA_ARCH__
    return __float_as_uint(x);
#else
    uint32_t u;
    memcpy(&u, &x, sizeof u);
    return u;
#endif
}

// Bin of position (x, y), or -1 outside the binned area (no segment lies within max_range there).
__host__ __device__ __forceinline__ int obs_bin(const ObsParams &m, float x, float y)
{
    const float fx = (x - m.bx0) * m.inv_bin, fy = (y - m.by0) * m.inv_bin;
    if (!(fx >= 0.0f && fx < (float)m.nbx && fy >= 0.0f && fy < (float)m.nby)) return -1;
    const int ix = (int)fx, iy = (int)fy;
    return (iy < m.nby - 1 ? iy : m.nby - 1) * m.nbx + (ix < m.nbx - 1 ? ix : m.nbx - 1);
}

// Segment s is a candidate of agent a when its squared distance from the agent, d2, is below range^2 and the agent is
// strictly on its free (right) side.  d2: clamp t = -(r1 . e) / |e|^2 to [0, 1], d2 = |r1 + t e|^2 with r1 = s.x0 - a,
// e = s.x1 - s.x0, in float32; the sort key of the candidates is (d2, segment index).
__host__ __device__ __forceinline__ bool obs_candidate(const OrcaAgent &a, const ObsSeg &s, float range2, float &d2)
{
    const float r1x = s.x0 - a.px, r1y = s.y0 - a.py, ex = s.x1 - s.x0, ey = s.y1 - s.y0;
    const float t = fminf(fmaxf(-(r1x * ex + r1y * ey) / (ex * ex + ey * ey), 0.0f), 1.0f);
    const float qx = r1x + t * ex, qy = r1y + t * ey;
    d2 = qx * qx + qy * qy;
    return d2 < range2 && det2(s.dx, s.dy, -r1x, -r1y) < 0.0f;
}

// Segment s is covered by obstacle line l when both its vertices, scaled by 1 / tau_o, lie at least r_o / tau_o -
// OBS_COVER_EPS beyond l (on its forbidden side).  The tolerance is RVO2's: a cut-off arc line is tangent to the disk of
// radius r_o / tau_o round a vertex the next segment shares, so that vertex lies exactly r_o / tau_o beyond the line,
// and without it rounding alone would decide whether the next segment adds a copy of the same line.
#define OBS_COVER_EPS 1e-5f
__host__ __device__ __forceinline__ bool obs_covered(const OrcaLine &l, const OrcaAgent &a, const ObsSeg &s,
                                                     const ObsParams &m)
{
    const float ax = m.inv_tau * (s.x0 - a.px) - l.px, ay = m.inv_tau * (s.y0 - a.py) - l.py;
    const float bx = m.inv_tau * (s.x1 - a.px) - l.px, by = m.inv_tau * (s.y1 - a.py) - l.py;
    return det2(ax, ay, l.dx, l.dy) - m.rt >= -OBS_COVER_EPS && det2(bx, by, l.dx, l.dy) - m.rt >= -OBS_COVER_EPS;
}

__host__ __device__ __forceinline__ void obs_unit(float x, float y, float &ux, float &uy)
{
    const float n = sqrtf(x * x + y * y);
    ux = x / n;
    uy = y / n;
}

// Leg directions of the truncated velocity obstacle of the disk of radius r at relative position (x, y), d2 = x^2 + y^2
// > r^2: the tangents from the origin, left and right as seen from the agent.
__host__ __device__ __forceinline__ void obs_legs(float x, float y, float d2, float r, float &lx, float &ly, float &rx,
                                                  float &ry)
{
    const float leg = sqrtf(d2 - r * r);
    lx = (x * leg - y * r) / d2;
    ly = (x * r + y * leg) / d2;
    rx = (x * leg + y * r) / d2;
    ry = (-x * r + y * leg) / d2;
}

// The obstacle half-plane of segment s for agent a (RVO2's Agent::computeNewVelocity, obstacle part): the velocity
// obstacle of s grown by r_o with horizon tau_o is the cut-off segment (the edge / tau_o grown by r_o / tau_o) and two
// legs; a leg at a non-convex vertex runs along the segment, and a leg that points into the neighbouring segment
// (foreign) is replaced by that segment's direction.  The line is tangent to the obstacle at its boundary point nearest
// to the current velocity, through that point (full responsibility).  When the agent is closer than r_o to s the line
// passes through the origin, perpendicular to the direction to the nearest point.  False when s adds no line: a
// colliding non-convex end vertex, a vertex the neighbouring segment handles, or a nearest point on a foreign leg.
__host__ __device__ __forceinline__ bool obstacle_line(const OrcaAgent &a, const ObsSeg &s, const ObsParams &m,
                                                       OrcaLine &l)
{
    const float r = m.r, r2 = r * r;
    const float r1x = s.x0 - a.px, r1y = s.y0 - a.py, r2x = s.x1 - a.px, r2y = s.y1 - a.py;
    const float ex = s.x1 - s.x0, ey = s.y1 - s.y0;
    const float d1 = r1x * r1x + r1y * r1y, d2 = r2x * r2x + r2y * r2y;
    const float t = -(r1x * ex + r1y * ey) / (ex * ex + ey * ey);
    const float qx = -r1x - t * ex, qy = -r1y - t * ey, dline = qx * qx + qy * qy;
    if (t < 0.0f && d1 <= r2) {                     // collision with the start vertex
        if (!s.convex0) return false;
        l.px = 0.0f; l.py = 0.0f;
        obs_unit(-r1y, r1x, l.dx, l.dy);
        return true;
    }
    if (t > 1.0f && d2 <= r2) {                     // collision with the end vertex
        if (!s.convex1 || det2(r2x, r2y, s.ndx, s.ndy) < 0.0f) return false;
        l.px = 0.0f; l.py = 0.0f;
        obs_unit(-r2y, r2x, l.dx, l.dy);
        return true;
    }
    if (t >= 0.0f && t < 1.0f && dline <= r2) {     // collision with the segment
        l.px = 0.0f; l.py = 0.0f;
        l.dx = -s.dx; l.dy = -s.dy;
        return true;
    }
    // legs; `single` when one vertex alone shapes the obstacle (seen obliquely)
    float llx, lly, rlx, rly, c1x = r1x, c1y = r1y, c2x = r2x, c2y = r2y;
    float lnx = s.pdx, lny = s.pdy, rnx = s.ndx, rny = s.ndy;    // direction before the left / after the right vertex
    int lcv = s.convex0, rcv = s.convex1;
    bool single = false;
    if (t < 0.0f && dline <= r2) {
        if (!s.convex0) return false;
        single = true;
        c2x = r1x; c2y = r1y;
        rnx = s.dx; rny = s.dy; rcv = s.convex0;
        obs_legs(r1x, r1y, d1, r, llx, lly, rlx, rly);
    } else if (t > 1.0f && dline <= r2) {
        if (!s.convex1) return false;
        single = true;
        c1x = r2x; c1y = r2y;
        lnx = s.dx; lny = s.dy; lcv = s.convex1;
        obs_legs(r2x, r2y, d2, r, llx, lly, rlx, rly);
    } else {
        float ux, uy;
        if (s.convex0) obs_legs(r1x, r1y, d1, r, llx, lly, ux, uy);
        else { llx = -s.dx; lly = -s.dy; }
        if (s.convex1) obs_legs(r2x, r2y, d2, r, ux, uy, rlx, rly);
        else { rlx = s.dx; rly = s.dy; }
    }
    bool lforeign = false, rforeign = false;
    if (lcv && det2(llx, lly, -lnx, -lny) >= 0.0f) { llx = -lnx; lly = -lny; lforeign = true; }
    if (rcv && det2(rlx, rly, rnx, rny) <= 0.0f) { rlx = rnx; rly = rny; rforeign = true; }
    const float lcx = m.inv_tau * c1x, lcy = m.inv_tau * c1y, rcx = m.inv_tau * c2x, rcy = m.inv_tau * c2y;
    const float cvx = rcx - lcx, cvy = rcy - lcy;
    const float wlx = a.vx - lcx, wly = a.vy - lcy, wrx = a.vx - rcx, wry = a.vy - rcy;
    const float tc = single ? 0.5f : (wlx * cvx + wly * cvy) / (cvx * cvx + cvy * cvy);
    const float tl = wlx * llx + wly * lly, tr = wrx * rlx + wry * rly;
    if ((tc < 0.0f && tl < 0.0f) || (single && tl < 0.0f && tr < 0.0f)) {     // the left cut-off arc
        float ux, uy;
        obs_unit(wlx, wly, ux, uy);
        l.dx = uy; l.dy = -ux;
        l.px = lcx + m.rt * ux; l.py = lcy + m.rt * uy;
        return true;
    }
    if (tc > 1.0f && tr < 0.0f) {                                              // the right cut-off arc
        float ux, uy;
        obs_unit(wrx, wry, ux, uy);
        l.dx = uy; l.dy = -ux;
        l.px = rcx + m.rt * ux; l.py = rcy + m.rt * uy;
        return true;
    }
    float dc = INFINITY, dl = INFINITY, dr = INFINITY;
    if (!(tc < 0.0f || tc > 1.0f || single)) {
        const float x = wlx - tc * cvx, y = wly - tc * cvy;
        dc = x * x + y * y;
    }
    if (!(tl < 0.0f)) {
        const float x = wlx - tl * llx, y = wly - tl * lly;
        dl = x * x + y * y;
    }
    if (!(tr < 0.0f)) {
        const float x = wrx - tr * rlx, y = wry - tr * rly;
        dr = x * x + y * y;
    }
    float cx, cy;
    if (dc <= dl && dc <= dr) {                                                // the cut-off segment
        l.dx = -s.dx; l.dy = -s.dy; cx = lcx; cy = lcy;
    } else if (dl <= dr) {                                                     // the left leg
        if (lforeign) return false;
        l.dx = llx; l.dy = lly; cx = lcx; cy = lcy;
    } else {                                                                   // the right leg
        if (rforeign) return false;
        l.dx = -rlx; l.dy = -rly; cx = rcx; cy = rcy;
    }
    l.px = cx + m.rt * -l.dy;
    l.py = cy + m.rt * l.dx;
    return true;
}

// ------------------------------------------------------------------------------------ device: one warp per agent
__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fminf(v, __shfl_xor_sync(FULL_MASK, v, o));
    return v;
}

// 2-D LP over lines[0, n): returns the first line that makes it infeasible (the result is then the optimum of the lines
// before it), or n.  Every lane holds the same result.
__device__ int lp2_warp(const OrcaLine *lines, int n, float radius, float ox, float oy, bool dir_opt, float &rx,
                        float &ry, int lane)
{
    lp2_start(radius, ox, oy, dir_opt, rx, ry);
    for (int i = 0; i < n; ++i) {
        const OrcaLine li = lines[i];
        if (!violates(li, rx, ry)) continue;
        float tl, tr;
        bool ok = lp1_range(li, radius, tl, tr);
        if (ok) {
            float lo = -INFINITY, hi = INFINITY;
            bool bad = false;
            for (int k = lane; k < i; k += 32) {
                float b;
                const int kind = lp1_bound(li, lines[k], b);
                if (kind == 2) bad = true;
                else if (kind == 1) hi = fminf(hi, b);
                else if (kind == -1) lo = fmaxf(lo, b);
            }
            tl = fmaxf(tl, warp_max(lo));
            tr = fminf(tr, warp_min(hi));
            ok = !__any_sync(FULL_MASK, bad) && tl <= tr;
        }
        if (!ok) return i;
        lp1_pick(li, tl, tr, ox, oy, dir_opt, rx, ry);
    }
    return n;
}

// Least-penetration fallback from line `begin` on (the result holds the optimum of the lines before it).  Lines
// [0, hard) stay hard: they enter every projected LP unchanged, as RVO2's linearProgram3 keeps obstacle lines.
__device__ void lp3_warp(const OrcaLine *lines, int n, int begin, int hard, float radius, OrcaLine *proj, float &rx,
                         float &ry, int lane)
{
    float dist = 0.0f;
    for (int i = begin; i < n; ++i) {
        const OrcaLine li = lines[i];
        if (!(det2(li.dx, li.dy, li.px - rx, li.py - ry) > dist)) continue;
        int np = 0;
        for (int j0 = 0; j0 < i; j0 += 32) {
            const int j = j0 + lane;
            OrcaLine o;
            bool keep = false;
            if (j < i) {
                if (j < hard) {
                    o = lines[j];
                    keep = true;
                } else {
                    keep = lp3_line(li, lines[j], o);
                }
            }
            const unsigned m = __ballot_sync(FULL_MASK, keep);
            if (keep) proj[np + __popc(m & ((1u << lane) - 1u))] = o;
            np += __popc(m);
        }
        __syncwarp();
        const float sx = rx, sy = ry;
        if (lp2_warp(proj, np, radius, -li.dy, li.dx, true, rx, ry, lane) < np) { rx = sx; ry = sy; }
        dist = det2(li.dx, li.dy, li.px - rx, li.py - ry);
        __syncwarp();
    }
}

// The obstacle lines of agent a into out[0, return): the candidates of its bin (obs_candidate) are compacted into
// key[] as (d2 bits << 32 | segment index), ranked by counting (keys are distinct) into order[], and then taken in that
// order: a candidate covered by a line built so far (tested across the lanes, any-ballot) is skipped, else its line is
// built (every lane computes the same line; lane 0 stores it).  dropped = 1 when a line found no room among the
// OBS_LINES; the lines kept are then the nearest ones and processing stops.
__device__ int obs_lines_warp(const OrcaAgent &me, const ObsParams &m, OrcaLine *out, unsigned long long *key,
                              int32_t *order, int lane, int &dropped)
{
    const int bin = obs_bin(m, me.px, me.py);
    int nc = 0;
    if (bin >= 0) {
        const int b0 = m.bin_off[bin], b1 = m.bin_off[bin + 1];
        for (int k0 = b0; k0 < b1; k0 += 32) {
            const int k = k0 + lane;
            unsigned long long kk = 0ull;
            bool keep = false;
            if (k < b1) {
                const int si = m.bin_idx[k];
                float d2;
                keep = obs_candidate(me, m.seg[si], m.range2, d2);
                kk = ((unsigned long long)float_bits(d2) << 32) | (unsigned)si;
            }
            const unsigned msk = __ballot_sync(FULL_MASK, keep);
            if (keep) key[nc + __popc(msk & ((1u << lane) - 1u))] = kk;
            nc += __popc(msk);
        }
    }
    __syncwarp();
    for (int k = lane; k < nc; k += 32) {
        const unsigned long long kk = key[k];
        int rank = 0;
        for (int j = 0; j < nc; ++j) rank += key[j] < kk;
        order[rank] = (int32_t)(kk & 0xffffffffull);
    }
    __syncwarp();
    int no = 0;
    dropped = 0;
    for (int c = 0; c < nc; ++c) {
        const ObsSeg s = m.seg[order[c]];
        bool cov = false;
        for (int k = lane; k < no; k += 32) cov |= obs_covered(out[k], me, s, m);
        if (__any_sync(FULL_MASK, cov)) continue;
        OrcaLine l;
        if (!obstacle_line(me, s, m, l)) continue;
        if (no == OBS_LINES) { dropped = 1; break; }
        if (lane == 0) out[no] = l;
        ++no;
        __syncwarp();
    }
    __syncwarp();
    return no;
}

// Dynamic shared memory of rlca_orca_kernel<NH, true>: per warp OBS_CAND keys, then per warp OBS_CAND indices.
#define OBS_SMEM (ORCA_WARPS * OBS_CAND * (sizeof(unsigned long long) + sizeof(int32_t)))

// NH = false: ORCA-DD (h unused); NH = true: NH-ORCA, P's lines first in the list.  MAP = true: the obstacle lines of
// the static map next (om), hard in the fallback; status bits 1 and 2 as rlca_orca_action_map documents.
template <bool NH, bool MAP>
__global__ void __launch_bounds__(ORCA_THREADS) rlca_orca_kernel(int n, int R, OrcaParams q, NhParams h,
                                                                  const float4 *__restrict__ pose,
                                                                  const float4 *__restrict__ goal,
                                                                  const int4 *__restrict__ meta,
                                                                  float2 *__restrict__ action,
                                                                  float2 *__restrict__ velocity,
                                                                  int32_t *__restrict__ status, ObsParams om)
{
    constexpr int max_lines = (NH ? NH_MAX_LINES : ORCA_MAX_LINES) + (MAP ? OBS_LINES : 0);
    __shared__ OrcaLine s_lines[ORCA_WARPS][max_lines];
    __shared__ OrcaLine s_proj[ORCA_WARPS][max_lines];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int a = blockIdx.x * ORCA_WARPS + warp;
    if (a >= n) return;
    const int base = a - a % R;
    const OrcaAgent me = orca_agent(pose, goal, meta, a);
    OrcaLine *lines = s_lines[warp];
    int nl = 0;
    if (NH) {
        if (lane < h.nv) lines[lane] = nh_hard_line(me, h.edge[lane]);
        nl = h.nv;
    }
    int hard = NH ? h.nv : 0, dropped = 0;
    if (MAP) {
        extern __shared__ unsigned long long s_obs[];
        __syncwarp();
        nl += obs_lines_warp(me, om, lines + nl, s_obs + warp * OBS_CAND,
                             reinterpret_cast<int32_t *>(s_obs + ORCA_WARPS * OBS_CAND) + warp * OBS_CAND, lane,
                             dropped);
        hard = nl;
    }
    for (int r0 = 0; r0 < R; r0 += 32) {
        const int b = base + r0 + lane;
        OrcaLine l;
        bool keep = false;
        if (r0 + lane < R && b != a) {
            const OrcaAgent o = orca_agent(pose, goal, meta, b);
            keep = orca_in_range(me, o, q.nd2) && orca_line(me, o, q, l);
        }
        const unsigned m = __ballot_sync(FULL_MASK, keep);
        if (keep) lines[nl + __popc(m & ((1u << lane) - 1u))] = l;
        nl += __popc(m);
    }
    __syncwarp();
    float ox, oy, rx, ry;
    orca_pref(me, goal[a], q, ox, oy);
    const int fail = lp2_warp(lines, nl, q.v_max, ox, oy, false, rx, ry, lane);
    if (fail < nl) lp3_warp(lines, nl, fail, hard, q.v_max, s_proj[warp], rx, ry, lane);
    if (lane == 0) {
        action[a] = NH ? nh_track(me, rx, ry, q, h) : orca_track(me, rx, ry, q);
        if (velocity) velocity[a] = make_float2(rx, ry);
        // bit 1: the fallback started at an obstacle line (lines [P's vertex count, hard))
        if (status) status[a] = MAP ? (fail < nl) | (fail >= (NH ? h.nv : 0) && fail < hard) << 1 | dropped << 2
                                    : fail < nl;
    }
}

// ------------------------------------------------------------------------------------ host: the serial loops
static int lp2_host(const OrcaLine *lines, int n, float radius, float ox, float oy, bool dir_opt, float &rx, float &ry)
{
    lp2_start(radius, ox, oy, dir_opt, rx, ry);
    for (int i = 0; i < n; ++i) {
        const OrcaLine &li = lines[i];
        if (!violates(li, rx, ry)) continue;
        float tl, tr;
        if (!lp1_range(li, radius, tl, tr)) return i;
        for (int k = 0; k < i; ++k) {
            float b;
            const int kind = lp1_bound(li, lines[k], b);
            if (kind == 2) return i;
            if (kind == 1) tr = fminf(tr, b);
            else if (kind == -1) tl = fmaxf(tl, b);
            if (tl > tr) return i;
        }
        lp1_pick(li, tl, tr, ox, oy, dir_opt, rx, ry);
    }
    return n;
}

static void lp3_host(const OrcaLine *lines, int n, int begin, int hard, float radius, float &rx, float &ry)
{
    OrcaLine proj[ALL_MAX_LINES];
    float dist = 0.0f;
    for (int i = begin; i < n; ++i) {
        const OrcaLine &li = lines[i];
        if (!(det2(li.dx, li.dy, li.px - rx, li.py - ry) > dist)) continue;
        int np = 0;
        for (int j = 0; j < i; ++j) {
            if (j < hard) proj[np++] = lines[j];
            else if (lp3_line(li, lines[j], proj[np])) ++np;
        }
        const float sx = rx, sy = ry;
        if (lp2_host(proj, np, radius, -li.dy, li.dx, true, rx, ry) < np) { rx = sx; ry = sy; }
        dist = det2(li.dx, li.dy, li.px - rx, li.py - ry);
    }
}

static int check_args(const rlca_env_config *cfg, float radius, float neighbour_dist, float time_horizon,
                      float heading_gain, OrcaParams &q)
{
    if (!cfg) return rlca_set_err(RLCA_ERR_INVALID, "cfg is NULL");
    if (cfg->robots_per_world < 1 || cfg->robots_per_world > RLCA_MAX_ROBOTS_PER_WORLD || cfg->num_worlds < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "cfg has no robots");
    if (!(cfg->dt > 0.0f) || !(cfg->v_max > 0.0f)) return rlca_set_err(RLCA_ERR_INVALID, "cfg needs dt > 0 and v_max > 0");
    const float ps[4] = {radius, neighbour_dist, time_horizon, heading_gain};
    for (float p : ps)
        if (!(p > 0.0f && p < INFINITY))
            return rlca_set_err(RLCA_ERR_INVALID, "ORCA radius, neighbour_dist, time_horizon and heading_gain must be "
                                                  "finite and > 0");
    q.r = 2.0f * radius;
    q.nd2 = neighbour_dist * neighbour_dist;
    q.inv_tau = 1.0f / time_horizon;
    q.inv_dt = 1.0f / cfg->dt;
    q.v_max = cfg->v_max;
    q.w_min = cfg->w_min;
    q.w_max = cfg->w_max;
    q.gain = heading_gain;
    return RLCA_OK;
}

extern "C" int rlca_orca_action(const rlca_env_config *cfg, const rlca_env_state *state, float radius,
                                float neighbour_dist, float time_horizon, float heading_gain, float *action_dev,
                                float *velocity_dev, int32_t *status_dev, void *stream)
{
    OrcaParams q;
    int rc = check_args(cfg, radius, neighbour_dist, time_horizon, heading_gain, q);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->meta_dev || !action_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_action: state or action buffer is NULL");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const NhParams none = {};
    const ObsParams no_map = {};
    rlca_orca_kernel<false, false><<<(n + ORCA_WARPS - 1) / ORCA_WARPS, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
        n, cfg->robots_per_world, q, none, reinterpret_cast<const float4 *>(state->pose_dev),
        reinterpret_cast<const float4 *>(state->goal_dev), reinterpret_cast<const int4 *>(state->meta_dev),
        reinterpret_cast<float2 *>(action_dev), reinterpret_cast<float2 *>(velocity_dev), status_dev, no_map);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

// obs_lines_warp by serial loops (std::sort of the same distinct keys gives the same order).
static int obs_lines_host(const OrcaAgent &me, const ObsParams &m, OrcaLine *out, int &dropped)
{
    std::vector<unsigned long long> key;
    const int bin = obs_bin(m, me.px, me.py);
    if (bin >= 0)
        for (int k = m.bin_off[bin]; k < m.bin_off[bin + 1]; ++k) {
            const int si = m.bin_idx[k];
            float d2;
            if (obs_candidate(me, m.seg[si], m.range2, d2))
                key.push_back(((unsigned long long)float_bits(d2) << 32) | (unsigned)si);
        }
    std::sort(key.begin(), key.end());
    int no = 0;
    dropped = 0;
    for (unsigned long long kk : key) {
        const ObsSeg &s = m.seg[(int32_t)(kk & 0xffffffffull)];
        bool cov = false;
        for (int k = 0; k < no && !cov; ++k) cov = obs_covered(out[k], me, s, m);
        if (cov) continue;
        OrcaLine l;
        if (!obstacle_line(me, s, m, l)) continue;
        if (no == OBS_LINES) { dropped = 1; break; }
        out[no++] = l;
    }
    return no;
}

// The per-agent steps of rlca_orca_kernel<NH, MAP> by serial loops; h = NULL is ORCA-DD, om = NULL map-blind.
static void host_actions(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                         const int32_t *meta_host, const OrcaParams &q, const NhParams *h, const ObsParams *om,
                         float *action_host, float *velocity_host, int32_t *status_host)
{
    const float4 *pose = reinterpret_cast<const float4 *>(pose_host), *goal = reinterpret_cast<const float4 *>(goal_host);
    const int4 *meta = reinterpret_cast<const int4 *>(meta_host);
    const int R = cfg->robots_per_world, n = R * cfg->num_worlds, nv = h ? h->nv : 0;
    OrcaLine lines[ALL_MAX_LINES];
    for (int a = 0; a < n; ++a) {
        const int base = a - a % R;
        const OrcaAgent me = orca_agent(pose, goal, meta, a);
        int nl = 0, hard = nv, dropped = 0;
        for (; nl < nv; ++nl) lines[nl] = nh_hard_line(me, h->edge[nl]);
        if (om) {
            nl += obs_lines_host(me, *om, lines + nl, dropped);
            hard = nl;
        }
        for (int b = base; b < base + R; ++b) {
            if (b == a) continue;
            const OrcaAgent o = orca_agent(pose, goal, meta, b);
            if (orca_in_range(me, o, q.nd2) && orca_line(me, o, q, lines[nl])) ++nl;
        }
        float ox, oy, rx, ry;
        orca_pref(me, goal[a], q, ox, oy);
        const int fail = lp2_host(lines, nl, q.v_max, ox, oy, false, rx, ry);
        if (fail < nl) lp3_host(lines, nl, fail, hard, q.v_max, rx, ry);
        const float2 act = h ? nh_track(me, rx, ry, q, *h) : orca_track(me, rx, ry, q);
        action_host[2 * a] = act.x;
        action_host[2 * a + 1] = act.y;
        if (velocity_host) { velocity_host[2 * a] = rx; velocity_host[2 * a + 1] = ry; }
        if (status_host)
            status_host[a] = om ? (fail < nl) | (fail >= nv && fail < hard) << 1 | dropped << 2 : fail < nl;
    }
}

extern "C" int rlca_orca_action_host(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                                     const int32_t *meta_host, float radius, float neighbour_dist, float time_horizon,
                                     float heading_gain, float *action_host, float *velocity_host, int32_t *status_host)
{
    OrcaParams q;
    int rc = check_args(cfg, radius, neighbour_dist, time_horizon, heading_gain, q);
    if (rc) return rc;
    if (!pose_host || !goal_host || !meta_host || !action_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_action_host: a buffer is NULL");
    host_actions(cfg, pose_host, goal_host, meta_host, q, nullptr, nullptr, action_host, velocity_host, status_host);
    return RLCA_OK;
}

// ------------------------------------------------------------------------------------ non-cooperative driver (§9h)
// ORCA-DD's action for agent a when it has no neighbours: v_pref on the speed disk, then the heading tracker.
__host__ __device__ __forceinline__ float2 noncoop_action(const float4 *pose, const float4 *goal, const int4 *meta, int a,
                                                          const OrcaParams &q)
{
    const OrcaAgent me = orca_agent(pose, goal, meta, a);
    float ox, oy, rx, ry;
    orca_pref(me, goal[a], q, ox, oy);
    lp2_start(q.v_max, ox, oy, false, rx, ry);
    return orca_track(me, rx, ry, q);
}

// One thread per agent; rows with mask 0 are not touched.
__global__ void __launch_bounds__(ORCA_THREADS) rlca_noncoop_kernel(int n, OrcaParams q,
                                                                     const float4 *__restrict__ pose,
                                                                     const float4 *__restrict__ goal,
                                                                     const int4 *__restrict__ meta,
                                                                     const uint8_t *__restrict__ mask,
                                                                     float2 *__restrict__ action)
{
    const int a = blockIdx.x * ORCA_THREADS + threadIdx.x;
    if (a >= n || !mask[a]) return;
    action[a] = noncoop_action(pose, goal, meta, a, q);
}

// ORCA-DD's parameters with v_max = speed and gain = heading_gain (the neighbour terms are unused).
static int noncoop_args(const rlca_env_config *cfg, float speed, float heading_gain, OrcaParams &q)
{
    if (!(heading_gain > 0.0f && heading_gain < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "non-cooperative heading_gain must be finite and > 0");
    int rc = check_args(cfg, 1.0f, 1.0f, 1.0f, heading_gain, q);
    if (rc) return rc;
    if (!(speed > 0.0f && speed <= cfg->v_max && speed < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "non-cooperative speed must be finite and in (0, cfg.v_max]");
    q.v_max = speed;
    return RLCA_OK;
}

extern "C" int rlca_noncoop_action(const rlca_env_config *cfg, const rlca_env_state *state, const uint8_t *mask_dev,
                                   float speed, float heading_gain, float *action_dev, void *stream)
{
    OrcaParams q;
    int rc = noncoop_args(cfg, speed, heading_gain, q);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->meta_dev || !mask_dev || !action_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_noncoop_action: state, mask or action buffer is NULL");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    rlca_noncoop_kernel<<<(n + ORCA_THREADS - 1) / ORCA_THREADS, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
        n, q, reinterpret_cast<const float4 *>(state->pose_dev), reinterpret_cast<const float4 *>(state->goal_dev),
        reinterpret_cast<const int4 *>(state->meta_dev), mask_dev, reinterpret_cast<float2 *>(action_dev));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_noncoop_action_host(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                                        const int32_t *meta_host, const uint8_t *mask_host, float speed,
                                        float heading_gain, float *action_host)
{
    OrcaParams q;
    int rc = noncoop_args(cfg, speed, heading_gain, q);
    if (rc) return rc;
    if (!pose_host || !goal_host || !meta_host || !mask_host || !action_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_noncoop_action_host: a buffer is NULL");
    const float4 *pose = reinterpret_cast<const float4 *>(pose_host), *goal = reinterpret_cast<const float4 *>(goal_host);
    const int4 *meta = reinterpret_cast<const int4 *>(meta_host);
    const int n = cfg->robots_per_world * cfg->num_worlds;
    for (int a = 0; a < n; ++a) {
        if (!mask_host[a]) continue;
        const float2 act = noncoop_action(pose, goal, meta, a, q);
        action_host[2 * a] = act.x;
        action_host[2 * a + 1] = act.y;
    }
    return RLCA_OK;
}

// ------------------------------------------------------------------------------------ hybrid controller (§9j)
// The scan minimum d (metres) of frame 2 of the stack picks the mode: 1 = the §9h driver at v_max when d > r_safe,
// 2 = the policy's action with v capped at v_safe when d < r_risk, 0 = the policy's action otherwise.
#define HYBRID_MODES 3

struct HybridParams {
    float r_safe, r_risk, v_safe, range_max;
};

__host__ __device__ __forceinline__ int hybrid_mode(float scan_min, const HybridParams &h)
{
    const float d = (scan_min + 0.5f) * h.range_max;
    return d > h.r_safe ? 1 : d < h.r_risk ? 2 : 0;
}

// Agent a's action for `mode`, in place; the count of the mode goes up when the tick belongs to a tracked episode.
__host__ __device__ __forceinline__ void hybrid_apply(int mode, const float4 *pose, const float4 *goal, const int4 *meta,
                                                      int a, const OrcaParams &q, const HybridParams &h,
                                                      const int32_t *open, float2 *action, uint8_t *mode_out,
                                                      int32_t *counts)
{
    if (mode == 1) action[a] = noncoop_action(pose, goal, meta, a, q);
    else if (mode == 2) action[a].x = fminf(action[a].x, h.v_safe);
    mode_out[a] = (uint8_t)mode;
    if (counts && open[a]) ++counts[(size_t)a * HYBRID_MODES + mode];
}

// One warp per agent: the lanes read beams lane, lane + 32, ... of frame 2 and take a shuffle minimum (exact and
// order-free, so it equals the host's serial loop); lane 0 picks the mode and writes.
__global__ void __launch_bounds__(ORCA_THREADS) rlca_hybrid_kernel(int n, int beams, OrcaParams q, HybridParams h,
                                                                    const float4 *__restrict__ pose,
                                                                    const float4 *__restrict__ goal,
                                                                    const int4 *__restrict__ meta,
                                                                    const float *__restrict__ stack,
                                                                    const int32_t *__restrict__ open,
                                                                    float2 *__restrict__ action,
                                                                    uint8_t *__restrict__ mode,
                                                                    int32_t *__restrict__ counts)
{
    const int a = blockIdx.x * ORCA_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (a >= n) return;
    const float *scan = stack + ((size_t)a * 3 + 2) * beams;
    float m = INFINITY;
    for (int k = lane; k < beams; k += 32) m = fminf(m, __ldg(scan + k));
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fminf(m, __shfl_xor_sync(FULL_MASK, m, o));
    if (lane == 0) hybrid_apply(hybrid_mode(m, h), pose, goal, meta, a, q, h, open, action, mode, counts);
}

static int hybrid_args(const rlca_env_config *cfg, const rlca_hybrid_params *p, OrcaParams &q, HybridParams &h)
{
    if (!cfg || !p) return rlca_set_err(RLCA_ERR_INVALID, "hybrid: cfg or params is NULL");
    if (cfg->beams < 1) return rlca_set_err(RLCA_ERR_INVALID, "hybrid: cfg has no beams");
    const float rm = cfg->range_max;
    if (!(p->r_risk >= 0.0f && p->r_risk <= p->r_safe && p->r_safe <= rm && rm < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "hybrid: need 0 <= r_risk <= r_safe <= cfg.range_max, all finite");
    if (!(p->heading_gain > 0.0f && p->heading_gain < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "hybrid: heading_gain must be finite and > 0");
    int rc = noncoop_args(cfg, cfg->v_max, p->heading_gain, q);
    if (rc) return rc;
    if (!(p->v_safe > 0.0f && p->v_safe <= cfg->v_max))
        return rlca_set_err(RLCA_ERR_INVALID, "hybrid: v_safe must be in (0, cfg.v_max]");
    h.r_safe = p->r_safe;
    h.r_risk = p->r_risk;
    h.v_safe = p->v_safe;
    h.range_max = rm;
    return RLCA_OK;
}

extern "C" int rlca_hybrid_action(const rlca_env_config *cfg, const rlca_hybrid_params *params,
                                  const rlca_env_state *state, const float *stack_dev, const int32_t *open_dev,
                                  float *action_dev, uint8_t *mode_dev, int32_t *counts_dev, void *stream)
{
    OrcaParams q;
    HybridParams h;
    int rc = hybrid_args(cfg, params, q, h);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->meta_dev || !stack_dev || !action_dev || !mode_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_hybrid_action: state, stack, action or mode buffer is NULL");
    if (!open_dev != !counts_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_hybrid_action: open and counts must be both set or both NULL");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    rlca_hybrid_kernel<<<(n + ORCA_WARPS - 1) / ORCA_WARPS, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
        n, cfg->beams, q, h, reinterpret_cast<const float4 *>(state->pose_dev),
        reinterpret_cast<const float4 *>(state->goal_dev), reinterpret_cast<const int4 *>(state->meta_dev), stack_dev,
        open_dev, reinterpret_cast<float2 *>(action_dev), mode_dev, counts_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_hybrid_action_host(const rlca_env_config *cfg, const rlca_hybrid_params *params,
                                       const float *stack_host, const float *pose_host, const float *goal_host,
                                       const int32_t *meta_host, const int32_t *open_host, float *action_host,
                                       uint8_t *mode_host, int32_t *counts_host)
{
    OrcaParams q;
    HybridParams h;
    int rc = hybrid_args(cfg, params, q, h);
    if (rc) return rc;
    if (!stack_host || !pose_host || !goal_host || !meta_host || !action_host || !mode_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_hybrid_action_host: a buffer is NULL");
    if (!open_host != !counts_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_hybrid_action_host: open and counts must be both set or both NULL");
    const float4 *pose = reinterpret_cast<const float4 *>(pose_host), *goal = reinterpret_cast<const float4 *>(goal_host);
    const int4 *meta = reinterpret_cast<const int4 *>(meta_host);
    const int n = cfg->robots_per_world * cfg->num_worlds, beams = cfg->beams;
    for (int a = 0; a < n; ++a) {
        const float *scan = stack_host + ((size_t)a * 3 + 2) * beams;
        float m = INFINITY;
        for (int k = 0; k < beams; ++k) m = fminf(m, scan[k]);
        hybrid_apply(hybrid_mode(m, h), pose, goal, meta, a, q, h, open_host, reinterpret_cast<float2 *>(action_host),
                     mode_host, counts_host);
    }
    return RLCA_OK;
}

// ------------------------------------------------------------------------------------ NH-ORCA: the velocity set P
struct NhSpec {
    double E, T, v_max, w_min, w_max;
};

// T_th, the arc tracker's turn time at angle th from the heading.
static double nh_turn_time(const NhSpec &s, double th) { return fmax(s.T, th / (th >= 0.0 ? s.w_max : s.w_min)); }

// V_max(th) = min(v_max, E / (T_th |sin(th / 2)|)): the largest speed at angle th whose tracking error is at most E.
static double nh_speed_bound(const NhSpec &s, double th)
{
    const double h = fabs(sin(0.5 * th));
    return h > 0.0 ? fmin(s.v_max, s.E / (nh_turn_time(s, th) * h)) : s.v_max;
}

// |v| / V_max(angle of v), at most 1 inside S_E.  On the negative x axis both sides of the cusp count.
static double nh_excess(const NhSpec &s, double x, double y)
{
    const double r = hypot(x, y);
    if (r == 0.0) return 0.0;
    if (y == 0.0 && x < 0.0) return fmax(r / nh_speed_bound(s, M_PI), r / nh_speed_bound(s, -M_PI));
    return r / nh_speed_bound(s, atan2(y, x));
}

// Largest excess on the segment a -> b: the best of m + 1 evenly spaced points, with `refine` a ternary search between
// that point's neighbours, and the point where the segment crosses the negative x axis.
static double nh_edge_excess(const NhSpec &s, const double *a, const double *b, int m, bool refine)
{
    const double ex = b[0] - a[0], ey = b[1] - a[1];
    auto at = [&](double t) { return nh_excess(s, a[0] + t * ex, a[1] + t * ey); };
    int best = 0;
    double worst = -1.0;
    for (int i = 0; i <= m; ++i) {
        const double e = at((double)i / m);
        if (e > worst) { worst = e; best = i; }
    }
    if (refine) {
        double lo = fmax(0.0, (best - 1.0) / m), hi = fmin(1.0, (best + 1.0) / m);
        for (int it = 0; it < 80; ++it) {
            const double t1 = lo + (hi - lo) / 3.0, t2 = hi - (hi - lo) / 3.0;
            if (at(t1) < at(t2)) lo = t1;
            else hi = t2;
        }
        worst = fmax(worst, at(0.5 * (lo + hi)));
    }
    if ((a[1] > 0.0) != (b[1] > 0.0)) {
        const double t = a[1] / (a[1] - b[1]), x = a[0] + t * ex;
        if (x < 0.0) worst = fmax(worst, nh_excess(s, x, 0.0));
    }
    return worst;
}

static double cross3(const double *o, const double *a, const double *b)
{
    return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0]);
}

// 1 / the largest excess over the edges of the closed polygon p (n vertices)
static double nh_fit(const NhSpec &s, const std::vector<double> &p, int n, int m, bool refine)
{
    double worst = 0.0;
    for (int i = 0; i < n; ++i) worst = fmax(worst, nh_edge_excess(s, &p[2 * i], &p[2 * ((i + 1) % n)], m, refine));
    return 1.0 / worst;
}

#define NH_SAMPLES 4096     // boundary angles of S_E
#define NH_MARGIN 1e-5      // P ends this far (relative) inside S_E, so that its rounding to float stays inside

// P in float64: the convex hull of S_E's boundary at NH_SAMPLES angles, scaled radially into S_E; then the vertex whose
// removal loses the least area is dropped until NH_ORCA_VERTS remain (removing a vertex of a convex polygon only
// shrinks it); then P is scaled radially until an edge reaches S_E less NH_MARGIN.  Writes the counter-clockwise
// vertices and returns their count, or 0 when P does not contain the origin strictly.
static int nh_build_polygon(const NhSpec &s, float *verts)
{
    std::vector<double> pts(2 * NH_SAMPLES);
    std::vector<int> order(NH_SAMPLES), hull(2 * NH_SAMPLES);
    for (int k = 0; k < NH_SAMPLES; ++k) {
        const double th = -M_PI + 2.0 * M_PI * k / NH_SAMPLES, r = nh_speed_bound(s, th);
        pts[2 * k] = r * cos(th);
        pts[2 * k + 1] = r * sin(th);
        order[k] = k;
    }
    // monotone chain: lower hull left to right, upper hull right to left
    std::sort(order.begin(), order.end(), [&](int i, int j) {
        return pts[2 * i] < pts[2 * j] || (pts[2 * i] == pts[2 * j] && pts[2 * i + 1] < pts[2 * j + 1]);
    });
    int k = 0;
    for (int i = 0; i < NH_SAMPLES; ++i) {
        while (k >= 2 && cross3(&pts[2 * hull[k - 2]], &pts[2 * hull[k - 1]], &pts[2 * order[i]]) <= 0.0) --k;
        hull[k++] = order[i];
    }
    for (int i = NH_SAMPLES - 2, lower = k + 1; i >= 0; --i) {
        while (k >= lower && cross3(&pts[2 * hull[k - 2]], &pts[2 * hull[k - 1]], &pts[2 * order[i]]) <= 0.0) --k;
        hull[k++] = order[i];
    }
    const int nh = k - 1;   // the last point repeats the first
    std::vector<double> H(2 * nh);
    for (int i = 0; i < nh; ++i) { H[2 * i] = pts[2 * hull[i]]; H[2 * i + 1] = pts[2 * hull[i] + 1]; }
    const double f0 = nh_fit(s, H, nh, 8, false);
    for (double &v : H) v *= f0;

    std::vector<int> prev(nh), next(nh);
    std::vector<double> loss(nh);
    std::vector<char> alive(nh, 1);
    auto tri = [&](int i) { return fabs(cross3(&H[2 * prev[i]], &H[2 * i], &H[2 * next[i]])); };
    for (int i = 0; i < nh; ++i) { prev[i] = (i + nh - 1) % nh; next[i] = (i + 1) % nh; }
    for (int i = 0; i < nh; ++i) loss[i] = tri(i);
    int first = 0;
    for (int left = nh; left > NH_ORCA_VERTS; --left) {
        int m = -1;
        for (int i = 0; i < nh; ++i)
            if (alive[i] && (m < 0 || loss[i] < loss[m])) m = i;
        alive[m] = 0;
        next[prev[m]] = next[m];
        prev[next[m]] = prev[m];
        loss[prev[m]] = tri(prev[m]);
        loss[next[m]] = tri(next[m]);
        if (m == first) first = next[m];
    }
    std::vector<double> P;
    int i = first;
    do {
        P.push_back(H[2 * i]);
        P.push_back(H[2 * i + 1]);
        i = next[i];
    } while (i != first);
    const int nv = (int)P.size() / 2;
    const double f1 = nh_fit(s, P, nv, 1024, true) * (1.0 - NH_MARGIN);
    for (int i = 0; i < 2 * nv; ++i) verts[i] = (float)(P[i] * f1);
    const double o[2] = {0.0, 0.0};
    for (int i = 0; i < nv; ++i) {
        const int j = (i + 1) % nv;
        const double a[2] = {verts[2 * i], verts[2 * i + 1]}, b[2] = {verts[2 * j], verts[2 * j + 1]};
        if (!(cross3(a, b, o) > 0.0)) return 0;
    }
    return nv;
}

// P for (E, T) and the config's bounds; the last one built is kept, since a controller asks for the same P every tick.
static int nh_polygon(const rlca_env_config *cfg, float tracking_error, float heading_time, float *verts, int &nv)
{
    struct Cache {
        float key[5];
        int nv;                                 // -1: empty
        float verts[2 * NH_ORCA_VERTS];
    };
    static thread_local Cache c = {{0.0f, 0.0f, 0.0f, 0.0f, 0.0f}, -1, {}};
    const float key[5] = {tracking_error, heading_time, cfg->v_max, cfg->w_min, cfg->w_max};
    if (c.nv < 0 || memcmp(key, c.key, sizeof key) != 0) {
        const NhSpec s = {tracking_error, heading_time, cfg->v_max, cfg->w_min, cfg->w_max};
        memcpy(c.key, key, sizeof key);
        c.nv = nh_build_polygon(s, c.verts);
    }
    if (c.nv == 0) return rlca_set_err(RLCA_ERR_INVALID, "NH-ORCA: the velocity polygon does not contain the origin");
    nv = c.nv;
    memcpy(verts, c.verts, 2 * nv * sizeof(float));
    return RLCA_OK;
}

static int nh_check_cfg(const rlca_env_config *cfg, float tracking_error, float heading_time)
{
    if (!cfg) return rlca_set_err(RLCA_ERR_INVALID, "cfg is NULL");
    if (!(cfg->v_min <= 0.0f && cfg->v_max > 0.0f && cfg->v_max < INFINITY && cfg->w_min < 0.0f &&
          cfg->w_min > -INFINITY && cfg->w_max > 0.0f && cfg->w_max < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "NH-ORCA needs cfg v_min <= 0 < v_max and w_min < 0 < w_max, finite");
    if (!(tracking_error > 0.0f && tracking_error < INFINITY && heading_time > 0.0f && heading_time < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "NH-ORCA tracking_error and heading_time must be finite and > 0");
    return RLCA_OK;
}

static int nh_check_args(const rlca_env_config *cfg, float radius, float neighbour_dist, float time_horizon,
                         float tracking_error, float heading_time, OrcaParams &q, NhParams &h)
{
    int rc = nh_check_cfg(cfg, tracking_error, heading_time);
    if (rc) return rc;
    const float ps[3] = {radius, neighbour_dist, time_horizon};
    for (float p : ps)
        if (!(p > 0.0f && p < INFINITY))
            return rlca_set_err(RLCA_ERR_INVALID, "NH-ORCA radius, neighbour_dist and time_horizon must be finite and "
                                                  "> 0");
    rc = check_args(cfg, radius, neighbour_dist, time_horizon, 1.0f, q);
    if (rc) return rc;
    q.r = 2.0f * (radius + tracking_error);
    float verts[2 * NH_ORCA_VERTS];
    memset(&h, 0, sizeof h);
    rc = nh_polygon(cfg, tracking_error, heading_time, verts, h.nv);
    if (rc) return rc;
    h.heading_time = heading_time;
    h.v_min = cfg->v_min;
    for (int k = 0; k < h.nv; ++k) {
        const int k1 = (k + 1) % h.nv;
        const double dx = (double)verts[2 * k1] - verts[2 * k], dy = (double)verts[2 * k1 + 1] - verts[2 * k + 1];
        const double l = sqrt(dx * dx + dy * dy);
        h.edge[k].px = verts[2 * k];
        h.edge[k].py = verts[2 * k + 1];
        h.edge[k].dx = (float)(dx / l);
        h.edge[k].dy = (float)(dy / l);
    }
    return RLCA_OK;
}

extern "C" int rlca_nh_orca_action(const rlca_env_config *cfg, const rlca_env_state *state, float radius,
                                   float neighbour_dist, float time_horizon, float tracking_error, float heading_time,
                                   float *action_dev, float *velocity_dev, int32_t *status_dev, void *stream)
{
    OrcaParams q;
    NhParams h;
    int rc = nh_check_args(cfg, radius, neighbour_dist, time_horizon, tracking_error, heading_time, q, h);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->meta_dev || !action_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_nh_orca_action: state or action buffer is NULL");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const ObsParams no_map = {};
    rlca_orca_kernel<true, false><<<(n + ORCA_WARPS - 1) / ORCA_WARPS, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
        n, cfg->robots_per_world, q, h, reinterpret_cast<const float4 *>(state->pose_dev),
        reinterpret_cast<const float4 *>(state->goal_dev), reinterpret_cast<const int4 *>(state->meta_dev),
        reinterpret_cast<float2 *>(action_dev), reinterpret_cast<float2 *>(velocity_dev), status_dev, no_map);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_nh_orca_action_host(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                                        const int32_t *meta_host, float radius, float neighbour_dist,
                                        float time_horizon, float tracking_error, float heading_time,
                                        float *action_host, float *velocity_host, int32_t *status_host)
{
    OrcaParams q;
    NhParams h;
    int rc = nh_check_args(cfg, radius, neighbour_dist, time_horizon, tracking_error, heading_time, q, h);
    if (rc) return rc;
    if (!pose_host || !goal_host || !meta_host || !action_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_nh_orca_action_host: a buffer is NULL");
    host_actions(cfg, pose_host, goal_host, meta_host, q, &h, nullptr, action_host, velocity_host, status_host);
    return RLCA_OK;
}

extern "C" int rlca_nh_orca_polygon_host(const rlca_env_config *cfg, float tracking_error, float heading_time,
                                         int32_t *nverts, float *verts_host)
{
    int rc = nh_check_cfg(cfg, tracking_error, heading_time);
    if (rc) return rc;
    if (!nverts || !verts_host) return rlca_set_err(RLCA_ERR_INVALID, "rlca_nh_orca_polygon_host: a buffer is NULL");
    int nv = 0;
    rc = nh_polygon(cfg, tracking_error, heading_time, verts_host, nv);
    if (rc) return rc;
    *nverts = nv;
    return RLCA_OK;
}

// ------------------------------------------------------------------------------------ static obstacles: the set (§9f)
struct rlca_orca_obstacles {
    std::vector<ObsSeg> seg;
    std::vector<int32_t> bin_off, bin_idx;
    float bx0, by0, max_range;
    int32_t nbx, nby, max_list;
    int device;                     // -1 until the device copy exists
    ObsSeg *seg_dev;
    int32_t *off_dev, *idx_dev;
};

// The boundary of the union of the occupied cells as closed loops, occupied cells on the left of every segment (loops
// run counter-clockwise round obstacles and clockwise round holes).  Unit cell edges are followed from corner to corner;
// at a corner where two occupied cells touch diagonally the loop turns right, so that it never passes between them
// (such cells count as connected).  Each segment is a maximal run of collinear unit edges.  Corner (i, j) lies at
// ((i - origin_cx) res, (j - origin_cy) res), computed in double and rounded to float once.
static int obs_build_segments(const uint8_t *cells, int W, int H, int ocx, int ocy, double res, std::vector<ObsSeg> &out)
{
    static const int DX[4] = {1, 0, -1, 0}, DY[4] = {0, 1, 0, -1};     // 0 +x, 1 +y, 2 -x, 3 -y; k + 1 turns left
    auto occ = [&](int i, int j) { return i >= 0 && j >= 0 && i < W && j < H && cells[(size_t)j * W + i] != 0; };
    // does a boundary edge leave corner (i, j) in direction k?  cells NE = (i, j), NW = (i-1, j), SW, SE
    auto leaves = [&](int i, int j, int k) {
        switch (k) {
        case 0: return occ(i, j) && !occ(i, j - 1);
        case 1: return occ(i - 1, j) && !occ(i, j);
        case 2: return occ(i - 1, j - 1) && !occ(i - 1, j);
        default: return occ(i, j - 1) && !occ(i - 1, j - 1);
        }
    };
    const size_t nh = (size_t)(H + 1) * W;
    auto edge_id = [&](int i, int j, int k) -> size_t {
        switch (k) {
        case 0: return (size_t)j * W + i;
        case 2: return (size_t)j * W + (i - 1);
        case 1: return nh + (size_t)j * (W + 1) + i;
        default: return nh + (size_t)(j - 1) * (W + 1) + i;
        }
    };
    std::vector<uint8_t> seen(nh + (size_t)H * (W + 1), 0);
    std::vector<int> ci, cj, dir;
    for (int j = 0; j < H; ++j)
        for (int i = 0; i < W; ++i) {
            if (!cells[(size_t)j * W + i]) continue;
            const int starts[4][3] = {{i, j, 0}, {i + 1, j, 1}, {i + 1, j + 1, 2}, {i, j + 1, 3}};
            for (const auto &st : starts) {
                if (!leaves(st[0], st[1], st[2]) || seen[edge_id(st[0], st[1], st[2])]) continue;
                ci.clear(); cj.clear(); dir.clear();
                int x = st[0], y = st[1], k = st[2];
                do {
                    seen[edge_id(x, y, k)] = 1;
                    ci.push_back(x); cj.push_back(y); dir.push_back(k);
                    x += DX[k]; y += DY[k];
                    const int turn[3] = {(k + 3) & 3, k, (k + 1) & 3};     // right, straight, left
                    int nk = -1;
                    for (int c : turn)
                        if (leaves(x, y, c)) { nk = c; break; }
                    if (nk < 0) return rlca_set_err(RLCA_ERR_INVALID, "obstacle boundary: open loop");
                    k = nk;
                } while (!(x == st[0] && y == st[1] && k == st[2]));
                const int n = (int)dir.size();
                int s0 = 0;
                while (dir[s0] == dir[(s0 + n - 1) % n]) ++s0;              // a corner: every loop turns
                const int first = (int)out.size();
                for (int e = 0; e < n;) {
                    const int a = (s0 + e) % n;
                    int len = 1;
                    while (e + len < n && dir[(s0 + e + len) % n] == dir[a]) ++len;
                    ObsSeg s = {};
                    s.x0 = (float)((ci[a] - ocx) * res);
                    s.y0 = (float)((cj[a] - ocy) * res);
                    s.x1 = (float)((ci[a] + len * DX[dir[a]] - ocx) * res);
                    s.y1 = (float)((cj[a] + len * DY[dir[a]] - ocy) * res);
                    s.dx = (float)DX[dir[a]];
                    s.dy = (float)DY[dir[a]];
                    s.convex0 = dir[a] == ((dir[(a + n - 1) % n] + 1) & 3);  // a left turn into the segment
                    out.push_back(s);
                    e += len;
                }
                const int last = (int)out.size() - 1;
                for (int s = first; s <= last; ++s) {
                    ObsSeg &g = out[s];
                    g.prev = s == first ? last : s - 1;
                    g.next = s == last ? first : s + 1;
                }
                for (int s = first; s <= last; ++s) {
                    ObsSeg &g = out[s];
                    g.pdx = out[g.prev].dx; g.pdy = out[g.prev].dy;
                    g.ndx = out[g.next].dx; g.ndy = out[g.next].dy;
                    g.convex1 = out[g.next].convex0;
                }
            }
        }
    return RLCA_OK;
}

// Bins of OBS_BIN m over the grid's extent grown by max_range + OBS_SLACK (rounded up to whole bins); a bin's list
// holds, in index order, every segment whose box is within max_range + OBS_SLACK of the bin's square.  An agent
// outside the binned area is farther than max_range from every segment.
static int obs_build_bins(rlca_orca_obstacles &o, int W, int H, int ocx, int ocy, double res)
{
    const double reach = (double)o.max_range + OBS_SLACK, margin = ceil(reach / OBS_BIN) * OBS_BIN;
    const double x0 = -ocx * res - margin, y0 = -ocy * res - margin;
    const double nbx = ceil((W * res + 2.0 * margin) / OBS_BIN), nby = ceil((H * res + 2.0 * margin) / OBS_BIN);
    if (nbx * nby > 1e8) return rlca_set_err(RLCA_ERR_UNSUPPORTED, "ORCA obstacles: too many lookup bins");
    o.bx0 = (float)x0;
    o.by0 = (float)y0;
    o.nbx = (int32_t)nbx;
    o.nby = (int32_t)nby;
    const size_t nb = (size_t)o.nbx * o.nby;
    std::vector<int32_t> count(nb + 1, 0);
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1) {
            o.bin_off.assign(nb + 1, 0);
            for (size_t b = 0; b < nb; ++b) o.bin_off[b + 1] = o.bin_off[b] + count[b];
            o.bin_idx.assign(o.bin_off[nb], 0);
            std::fill(count.begin(), count.end(), 0);
        }
        for (int si = 0; si < (int)o.seg.size(); ++si) {
            const ObsSeg &s = o.seg[si];
            const double lx = fmin(s.x0, s.x1), hx = fmax(s.x0, s.x1), ly = fmin(s.y0, s.y1), hy = fmax(s.y0, s.y1);
            const int ix0 = std::max(0, (int)floor((lx - reach - o.bx0) / OBS_BIN));
            const int ix1 = std::min(o.nbx - 1, (int)floor((hx + reach - o.bx0) / OBS_BIN));
            const int iy0 = std::max(0, (int)floor((ly - reach - o.by0) / OBS_BIN));
            const int iy1 = std::min(o.nby - 1, (int)floor((hy + reach - o.by0) / OBS_BIN));
            for (int iy = iy0; iy <= iy1; ++iy)
                for (int ix = ix0; ix <= ix1; ++ix) {
                    const double bx = (double)o.bx0 + ix * OBS_BIN, by = (double)o.by0 + iy * OBS_BIN;
                    const double gx = fmax(0.0, fmax(lx - (bx + OBS_BIN), bx - hx));
                    const double gy = fmax(0.0, fmax(ly - (by + OBS_BIN), by - hy));
                    if (gx * gx + gy * gy >= reach * reach) continue;
                    const size_t b = (size_t)iy * o.nbx + ix;
                    if (pass == 1) o.bin_idx[o.bin_off[b] + count[b]] = si;
                    ++count[b];
                }
        }
    }
    o.max_list = 0;
    for (size_t b = 0; b < nb; ++b) o.max_list = std::max(o.max_list, o.bin_off[b + 1] - o.bin_off[b]);
    if (o.max_list > OBS_CAND) {
        char msg[160];      // rlca_set_err formats string arguments only
        snprintf(msg, sizeof msg, "%d segments within max_range of one lookup bin, above RLCA_ORCA_MAP_MAX_CANDIDATES "
                 "= %d: lower max_range", o.max_list, OBS_CAND);
        return rlca_set_err(RLCA_ERR_UNSUPPORTED, "ORCA obstacles: %s", msg);
    }
    return RLCA_OK;
}

static void obs_free_device(rlca_orca_obstacles *o)
{
    if (o->device < 0) return;
    int cur = 0;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != o->device) cudaSetDevice(o->device);
    cudaFree(o->seg_dev);
    cudaFree(o->off_dev);
    cudaFree(o->idx_dev);
    if (cur != o->device) cudaSetDevice(cur);
    o->device = -1;
}

// The device copy, made on the current device; an obstacle set serves one device.
static int obs_device(rlca_orca_obstacles *o)
{
    int cur = 0;
    RLCA_CUDA_TRY(cudaGetDevice(&cur));
    if (o->device >= 0) {
        if (cur != o->device) return rlca_set_err(RLCA_ERR_INVALID, "ORCA obstacles: the set lives on another device");
        return RLCA_OK;
    }
    o->seg_dev = nullptr;
    o->off_dev = o->idx_dev = nullptr;
    o->device = cur;
    const size_t ns = std::max<size_t>(o->seg.size(), 1), no = o->bin_off.size(), ni = std::max<size_t>(o->bin_idx.size(), 1);
    cudaError_t e = cudaMalloc(&o->seg_dev, ns * sizeof(ObsSeg));
    if (e == cudaSuccess) e = cudaMalloc(&o->off_dev, no * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc(&o->idx_dev, ni * sizeof(int32_t));
    if (e == cudaSuccess && !o->seg.empty())
        e = cudaMemcpy(o->seg_dev, o->seg.data(), o->seg.size() * sizeof(ObsSeg), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(o->off_dev, o->bin_off.data(), no * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && !o->bin_idx.empty())
        e = cudaMemcpy(o->idx_dev, o->bin_idx.data(), o->bin_idx.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        obs_free_device(o);
        return rlca_set_err(RLCA_ERR_CUDA, "ORCA obstacles: device copy failed: %s", cudaGetErrorString(e));
    }
    return RLCA_OK;
}

extern "C" int rlca_orca_obstacles_create(const rlca_env_config *cfg, const uint8_t *cells_host, int32_t grid_w,
                                          int32_t grid_h, float max_range, rlca_orca_obstacles **out)
{
    if (!out) return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacles_create: out is NULL");
    *out = nullptr;
    if (!cfg || !cells_host) return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacles_create: cfg or cells is NULL");
    if (grid_w < 1 || grid_h < 1) return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacles_create: empty grid");
    if (!(cfg->resolution > 0.0f && cfg->resolution < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacles_create: cfg resolution must be finite and > 0");
    if (!(max_range > 0.0f && max_range < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacles_create: max_range must be finite and > 0");
    rlca_orca_obstacles *o = new rlca_orca_obstacles();
    o->device = -1;
    o->max_range = max_range;
    const double res = cfg->resolution;
    int rc = obs_build_segments(cells_host, grid_w, grid_h, cfg->origin_cx, cfg->origin_cy, res, o->seg);
    if (!rc) rc = obs_build_bins(*o, grid_w, grid_h, cfg->origin_cx, cfg->origin_cy, res);
    int ndev = 0;
    if (!rc) {
        if (cudaGetDeviceCount(&ndev) != cudaSuccess) {
            cudaGetLastError();
            ndev = 0;
        }
        if (ndev > 0) rc = obs_device(o);
    }
    if (rc) {
        delete o;
        return rc;
    }
    *out = o;
    return RLCA_OK;
}

extern "C" int rlca_orca_obstacles_destroy(rlca_orca_obstacles *obs)
{
    if (!obs) return RLCA_OK;
    obs_free_device(obs);
    delete obs;
    return RLCA_OK;
}

extern "C" int rlca_orca_obstacles_segments(const rlca_orca_obstacles *obs, int32_t *nsegments, int32_t *max_list,
                                            float *points_host, int32_t *links_host)
{
    if (!obs || !nsegments) return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacles_segments: obs or nsegments is NULL");
    *nsegments = (int32_t)obs->seg.size();
    if (max_list) *max_list = obs->max_list;
    for (size_t s = 0; s < obs->seg.size(); ++s) {
        const ObsSeg &g = obs->seg[s];
        if (points_host) {
            points_host[4 * s] = g.x0; points_host[4 * s + 1] = g.y0;
            points_host[4 * s + 2] = g.x1; points_host[4 * s + 3] = g.y1;
        }
        if (links_host) {
            links_host[3 * s] = g.prev; links_host[3 * s + 1] = g.next; links_host[3 * s + 2] = g.convex0;
        }
    }
    return RLCA_OK;
}

// The set's segments and bins as a launch reads them; device = true takes (or makes) the device copy.
static int obs_bins(rlca_orca_obstacles *obs, bool device, ObsParams &m)
{
    if (device) {
        const int rc = obs_device(obs);
        if (rc) return rc;
    }
    m.seg = device ? obs->seg_dev : obs->seg.data();
    m.bin_off = device ? obs->off_dev : obs->bin_off.data();
    m.bin_idx = device ? obs->idx_dev : obs->bin_idx.data();
    m.bx0 = obs->bx0;
    m.by0 = obs->by0;
    m.inv_bin = (float)(1.0 / OBS_BIN);
    m.nbx = obs->nbx;
    m.nby = obs->nby;
    return RLCA_OK;
}

// The launch parameters for obstacle radius r_o and horizon tau_o; device = true takes (or makes) the device copy.
static int obs_params(rlca_orca_obstacles *obs, const rlca_env_config *cfg, float r_o, float obstacle_time_horizon,
                      bool device, ObsParams &m)
{
    if (!obs) return rlca_set_err(RLCA_ERR_INVALID, "ORCA obstacles: the obstacle set is NULL");
    if (!(obstacle_time_horizon > 0.0f && obstacle_time_horizon < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "ORCA obstacle_time_horizon must be finite and > 0");
    const float range = obstacle_time_horizon * cfg->v_max + r_o;
    if (!(range <= obs->max_range))
        return rlca_set_err(RLCA_ERR_INVALID, "ORCA obstacles: obstacle_time_horizon * v_max + obstacle radius exceeds "
                                              "the set's max_range");
    const int rc = obs_bins(obs, device, m);
    if (rc) return rc;
    m.range2 = range * range;
    m.inv_tau = 1.0f / obstacle_time_horizon;
    m.r = r_o;
    m.rt = r_o * m.inv_tau;
    return RLCA_OK;
}

// The map kernels' dynamic shared memory exceeds the default limit; the attribute is set once per device.
template <bool NH>
static int map_smem_attribute()
{
    static std::atomic<unsigned long long> done{0ull};
    int dev = 0;
    RLCA_CUDA_TRY(cudaGetDevice(&dev));
    const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
    if (bit && (done.load() & bit)) return RLCA_OK;
    RLCA_CUDA_TRY(cudaFuncSetAttribute(rlca_orca_kernel<NH, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)OBS_SMEM));
    done.fetch_or(bit);
    return RLCA_OK;
}

template <bool NH>
static int launch_map(const rlca_env_config *cfg, const rlca_env_state *state, const OrcaParams &q, const NhParams &h,
                      const ObsParams &m, float *action_dev, float *velocity_dev, int32_t *status_dev, void *stream)
{
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const int rc = map_smem_attribute<NH>();
    if (rc) return rc;
    rlca_orca_kernel<NH, true><<<(n + ORCA_WARPS - 1) / ORCA_WARPS, ORCA_THREADS, OBS_SMEM, (cudaStream_t)stream>>>(
        n, cfg->robots_per_world, q, h, reinterpret_cast<const float4 *>(state->pose_dev),
        reinterpret_cast<const float4 *>(state->goal_dev), reinterpret_cast<const int4 *>(state->meta_dev),
        reinterpret_cast<float2 *>(action_dev), reinterpret_cast<float2 *>(velocity_dev), status_dev, m);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_orca_action_map(const rlca_env_config *cfg, const rlca_env_state *state,
                                    rlca_orca_obstacles *obstacles, float radius, float neighbour_dist,
                                    float time_horizon, float heading_gain, float obstacle_time_horizon,
                                    float *action_dev, float *velocity_dev, int32_t *status_dev, void *stream)
{
    OrcaParams q;
    ObsParams m;
    int rc = check_args(cfg, radius, neighbour_dist, time_horizon, heading_gain, q);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->meta_dev || !action_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_action_map: state or action buffer is NULL");
    rc = obs_params(obstacles, cfg, radius, obstacle_time_horizon, true, m);
    if (rc) return rc;
    const NhParams none = {};
    return launch_map<false>(cfg, state, q, none, m, action_dev, velocity_dev, status_dev, stream);
}

extern "C" int rlca_orca_action_map_host(const rlca_env_config *cfg, rlca_orca_obstacles *obstacles,
                                         const float *pose_host, const float *goal_host, const int32_t *meta_host,
                                         float radius, float neighbour_dist, float time_horizon, float heading_gain,
                                         float obstacle_time_horizon, float *action_host, float *velocity_host,
                                         int32_t *status_host)
{
    OrcaParams q;
    ObsParams m;
    int rc = check_args(cfg, radius, neighbour_dist, time_horizon, heading_gain, q);
    if (rc) return rc;
    if (!pose_host || !goal_host || !meta_host || !action_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_action_map_host: a buffer is NULL");
    rc = obs_params(obstacles, cfg, radius, obstacle_time_horizon, false, m);
    if (rc) return rc;
    host_actions(cfg, pose_host, goal_host, meta_host, q, nullptr, &m, action_host, velocity_host, status_host);
    return RLCA_OK;
}

extern "C" int rlca_nh_orca_action_map(const rlca_env_config *cfg, const rlca_env_state *state,
                                       rlca_orca_obstacles *obstacles, float radius, float neighbour_dist,
                                       float time_horizon, float tracking_error, float heading_time,
                                       float obstacle_time_horizon, float *action_dev, float *velocity_dev,
                                       int32_t *status_dev, void *stream)
{
    OrcaParams q;
    NhParams h;
    ObsParams m;
    int rc = nh_check_args(cfg, radius, neighbour_dist, time_horizon, tracking_error, heading_time, q, h);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->meta_dev || !action_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_nh_orca_action_map: state or action buffer is NULL");
    rc = obs_params(obstacles, cfg, radius + tracking_error, obstacle_time_horizon, true, m);
    if (rc) return rc;
    return launch_map<true>(cfg, state, q, h, m, action_dev, velocity_dev, status_dev, stream);
}

extern "C" int rlca_nh_orca_action_map_host(const rlca_env_config *cfg, rlca_orca_obstacles *obstacles,
                                            const float *pose_host, const float *goal_host, const int32_t *meta_host,
                                            float radius, float neighbour_dist, float time_horizon,
                                            float tracking_error, float heading_time, float obstacle_time_horizon,
                                            float *action_host, float *velocity_host, int32_t *status_host)
{
    OrcaParams q;
    NhParams h;
    ObsParams m;
    int rc = nh_check_args(cfg, radius, neighbour_dist, time_horizon, tracking_error, heading_time, q, h);
    if (rc) return rc;
    if (!pose_host || !goal_host || !meta_host || !action_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_nh_orca_action_map_host: a buffer is NULL");
    rc = obs_params(obstacles, cfg, radius + tracking_error, obstacle_time_horizon, false, m);
    if (rc) return rc;
    host_actions(cfg, pose_host, goal_host, meta_host, q, &h, &m, action_host, velocity_host, status_host);
    return RLCA_OK;
}

extern "C" int rlca_orca_obstacle_lines_host(const rlca_env_config *cfg, rlca_orca_obstacles *obstacles,
                                             const float *pose_host, const float *goal_host, const int32_t *meta_host,
                                             int32_t agent, float obstacle_radius, float obstacle_time_horizon,
                                             int32_t *nlines, int32_t *dropped, float *lines_host)
{
    if (!cfg || !pose_host || !goal_host || !meta_host || !nlines || !dropped || !lines_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacle_lines_host: a pointer is NULL");
    if (agent < 0 || agent >= cfg->robots_per_world * cfg->num_worlds)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacle_lines_host: agent out of range");
    if (!(obstacle_radius > 0.0f && obstacle_radius < INFINITY) || !(cfg->v_max > 0.0f && cfg->v_max < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_orca_obstacle_lines_host: obstacle_radius and cfg v_max must be "
                                              "finite and > 0");
    ObsParams m;
    const int rc = obs_params(obstacles, cfg, obstacle_radius, obstacle_time_horizon, false, m);
    if (rc) return rc;
    const OrcaAgent me = orca_agent(reinterpret_cast<const float4 *>(pose_host),
                                    reinterpret_cast<const float4 *>(goal_host),
                                    reinterpret_cast<const int4 *>(meta_host), agent);
    OrcaLine lines[OBS_LINES];
    int d = 0;
    const int no = obs_lines_host(me, m, lines, d);
    for (int k = 0; k < no; ++k) {
        lines_host[4 * k] = lines[k].px; lines_host[4 * k + 1] = lines[k].py;
        lines_host[4 * k + 2] = lines[k].dx; lines_host[4 * k + 3] = lines[k].dy;
    }
    *nlines = no;
    *dropped = d;
    return RLCA_OK;
}

// ------------------------------------------------------------------------------------ social-force crowd (§9t)
// Masked agents steer by a Helbing-Molnar style social force: a driving term towards the §9h driver's preferred
// velocity, an anisotropic repulsion with a sideways bias from the other agents of the world, a repulsion from the
// static map's segments, and ORCA-DD's heading tracker on the velocity that results.
struct CrowdParams {
    float inv_relax, strength, range, aniso, side_bias, two_r, nd;
    float wall_strength, wall_range, radius, dt;
    int32_t see_robots;
};

// The force an agent at (ox, oy) exerts on me, added to (fx, fy); none unless 0 < d < neighbour_dist.
__host__ __device__ __forceinline__ void crowd_agent_force(const OrcaAgent &me, float ox, float oy,
                                                           const CrowdParams &c, float &fx, float &fy)
{
    const float dx = me.px - ox, dy = me.py - oy, d = sqrtf(dx * dx + dy * dy);
    if (!(d > 0.0f && d < c.nd)) return;
    const float nx = dx / d, ny = dy / d, tx = -ny, ty = nx;
    const float cphi = -(nx * me.ct + ny * me.st);
    const float w = c.aniso + (1.0f - c.aniso) * (1.0f + cphi) * 0.5f;
    const float k = c.strength * dev_expf((c.two_r - d) / c.range) * w;
    fx += k * (nx + c.side_bias * tx);
    fy += k * (ny + c.side_bias * ty);
}

// The force segment s exerts on me, added to (fx, fy), when it is a candidate (obs_candidate with m.range2 =
// wall_dist^2); q is its nearest point, computed as obs_candidate computes it.
__host__ __device__ __forceinline__ void crowd_wall_force(const OrcaAgent &me, const ObsSeg &s, const ObsParams &m,
                                                          const CrowdParams &c, float &fx, float &fy)
{
    float d2;
    if (!obs_candidate(me, s, m.range2, d2)) return;
    const float r1x = s.x0 - me.px, r1y = s.y0 - me.py, ex = s.x1 - s.x0, ey = s.y1 - s.y0;
    const float t = fminf(fmaxf(-(r1x * ex + r1y * ey) / (ex * ex + ey * ey), 0.0f), 1.0f);
    const float qx = r1x + t * ex, qy = r1y + t * ey, d = sqrtf(d2);
    if (!(d > 0.0f)) return;
    const float k = c.wall_strength * dev_expf((c.radius - d) / c.wall_range);
    fx += k * (-qx / d);
    fy += k * (-qy / d);
}

// The action from the summed agent and wall forces (sx, sy): driving term, one Euler step on the speed disk, tracker.
__host__ __device__ __forceinline__ float2 crowd_action(const OrcaAgent &me, float4 goal, const OrcaParams &q,
                                                        const CrowdParams &c, float sx, float sy)
{
    float ox, oy, ux, uy;
    orca_pref(me, goal, q, ox, oy);
    const float fx = (ox - me.vx) * c.inv_relax + sx, fy = (oy - me.vy) * c.inv_relax + sy;
    lp2_start(q.v_max, me.vx + fx * c.dt, me.vy + fy * c.dt, false, ux, uy);
    return orca_track(me, ux, uy, q);
}

// One warp per agent; warps of unmasked agents return at once.  Lane l sums the forces of agents base + l, l + 32, ...
// and then of bin entries b0 + l, b0 + l + 32, ..., in that order; the xor butterfly (offsets 16 .. 1) adds the
// partials, and every lane ends with the same sum since each step adds the same two values on both lanes of a pair.
template <bool MAP>
__global__ void __launch_bounds__(ORCA_THREADS) rlca_crowd_kernel(int n, int R, OrcaParams q, CrowdParams c,
                                                                   const float4 *__restrict__ pose,
                                                                   const float4 *__restrict__ goal,
                                                                   const int4 *__restrict__ meta,
                                                                   const uint8_t *__restrict__ mask,
                                                                   float2 *__restrict__ action, ObsParams om)
{
    const int a = blockIdx.x * ORCA_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (a >= n || !mask[a]) return;
    const int base = a - a % R;
    const OrcaAgent me = orca_agent(pose, goal, meta, a);
    float fx = 0.0f, fy = 0.0f;
    for (int j = lane; j < R; j += 32) {
        const int b = base + j;
        if (b != a && (c.see_robots || mask[b])) {
            const float4 p = pose[b];
            crowd_agent_force(me, p.x, p.y, c, fx, fy);
        }
    }
    if (MAP) {
        const int bin = obs_bin(om, me.px, me.py);
        if (bin >= 0)
            for (int k = om.bin_off[bin] + lane; k < om.bin_off[bin + 1]; k += 32)
                crowd_wall_force(me, om.seg[om.bin_idx[k]], om, c, fx, fy);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        fx += __shfl_xor_sync(FULL_MASK, fx, o);
        fy += __shfl_xor_sync(FULL_MASK, fy, o);
    }
    if (lane == 0) action[a] = crowd_action(me, goal[a], q, c, fx, fy);
}

static int crowd_args(const rlca_env_config *cfg, const rlca_crowd_params *p, const rlca_orca_obstacles *obs,
                      OrcaParams &q, CrowdParams &c)
{
    if (!cfg || !p) return rlca_set_err(RLCA_ERR_INVALID, "crowd: cfg or params is NULL");
    const float pos[6] = {p->relax_time, p->range, p->wall_range, p->radius, p->neighbour_dist, p->heading_gain};
    for (float x : pos)
        if (!(x > 0.0f && x < INFINITY))
            return rlca_set_err(RLCA_ERR_INVALID, "crowd: relax_time, range, wall_range, radius, neighbour_dist and "
                                                  "heading_gain must be finite and > 0");
    if (!(p->strength >= 0.0f && p->strength < INFINITY && p->wall_strength >= 0.0f && p->wall_strength < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "crowd: strength and wall_strength must be finite and >= 0");
    if (!(p->anisotropy >= 0.0f && p->anisotropy <= 1.0f))
        return rlca_set_err(RLCA_ERR_INVALID, "crowd: anisotropy must be in [0, 1]");
    if (!(p->side_bias >= 0.0f && p->side_bias < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "crowd: side_bias must be finite and >= 0");
    if (!(p->wall_dist > 0.0f && p->wall_dist < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "crowd: wall_dist must be finite and > 0");
    if (obs && !(p->wall_dist <= obs->max_range))
        return rlca_set_err(RLCA_ERR_INVALID, "crowd: wall_dist exceeds the obstacle set's max_range");
    if (!(p->speed > 0.0f && p->speed <= cfg->v_max && p->speed < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "crowd: speed must be finite and in (0, cfg.v_max]");
    const int rc = noncoop_args(cfg, p->speed, p->heading_gain, q);
    if (rc) return rc;
    c.inv_relax = 1.0f / p->relax_time;
    c.strength = p->strength;
    c.range = p->range;
    c.aniso = p->anisotropy;
    c.side_bias = p->side_bias;
    c.two_r = 2.0f * p->radius;
    c.nd = p->neighbour_dist;
    c.wall_strength = p->wall_strength;
    c.wall_range = p->wall_range;
    c.radius = p->radius;
    c.dt = cfg->dt;
    c.see_robots = p->see_robots != 0;
    return RLCA_OK;
}

extern "C" int rlca_crowd_action(const rlca_env_config *cfg, const rlca_crowd_params *params,
                                 const rlca_env_state *state, const uint8_t *mask_dev, rlca_orca_obstacles *obstacles,
                                 float *action_dev, void *stream)
{
    OrcaParams q;
    CrowdParams c;
    ObsParams m = {};
    int rc = crowd_args(cfg, params, obstacles, q, c);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->meta_dev || !mask_dev || !action_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_crowd_action: state, mask or action buffer is NULL");
    if (obstacles) {
        rc = obs_bins(obstacles, true, m);
        if (rc) return rc;
        m.range2 = params->wall_dist * params->wall_dist;
    }
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const dim3 grid((n + ORCA_WARPS - 1) / ORCA_WARPS);
    const float4 *pose = reinterpret_cast<const float4 *>(state->pose_dev);
    const float4 *goal = reinterpret_cast<const float4 *>(state->goal_dev);
    const int4 *meta = reinterpret_cast<const int4 *>(state->meta_dev);
    float2 *action = reinterpret_cast<float2 *>(action_dev);
    if (obstacles)
        rlca_crowd_kernel<true><<<grid, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
            n, cfg->robots_per_world, q, c, pose, goal, meta, mask_dev, action, m);
    else
        rlca_crowd_kernel<false><<<grid, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
            n, cfg->robots_per_world, q, c, pose, goal, meta, mask_dev, action, m);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

// rlca_crowd_kernel by serial loops: the 32 lanes' partials in the same order, then the same butterfly.
extern "C" int rlca_crowd_action_host(const rlca_env_config *cfg, const rlca_crowd_params *params,
                                      rlca_orca_obstacles *obstacles, const float *pose_host, const float *goal_host,
                                      const int32_t *meta_host, const uint8_t *mask_host, float *action_host)
{
    OrcaParams q;
    CrowdParams c;
    ObsParams m = {};
    int rc = crowd_args(cfg, params, obstacles, q, c);
    if (rc) return rc;
    if (!pose_host || !goal_host || !meta_host || !mask_host || !action_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_crowd_action_host: a buffer is NULL");
    if (obstacles) {
        rc = obs_bins(obstacles, false, m);
        if (rc) return rc;
        m.range2 = params->wall_dist * params->wall_dist;
    }
    const float4 *pose = reinterpret_cast<const float4 *>(pose_host), *goal = reinterpret_cast<const float4 *>(goal_host);
    const int4 *meta = reinterpret_cast<const int4 *>(meta_host);
    const int R = cfg->robots_per_world, n = R * cfg->num_worlds;
    for (int a = 0; a < n; ++a) {
        if (!mask_host[a]) continue;
        const int base = a - a % R;
        const OrcaAgent me = orca_agent(pose, goal, meta, a);
        float fx[32] = {}, fy[32] = {}, gx[32], gy[32];
        for (int j = 0; j < R; ++j) {
            const int b = base + j;
            if (b != a && (c.see_robots || mask_host[b]))
                crowd_agent_force(me, pose[b].x, pose[b].y, c, fx[j & 31], fy[j & 31]);
        }
        if (obstacles) {
            const int bin = obs_bin(m, me.px, me.py);
            if (bin >= 0)
                for (int k = m.bin_off[bin]; k < m.bin_off[bin + 1]; ++k)
                    crowd_wall_force(me, m.seg[m.bin_idx[k]], m, c, fx[(k - m.bin_off[bin]) & 31],
                                     fy[(k - m.bin_off[bin]) & 31]);
        }
        for (int o = 16; o; o >>= 1) {
            for (int l = 0; l < 32; ++l) { gx[l] = fx[l] + fx[l ^ o]; gy[l] = fy[l] + fy[l ^ o]; }
            memcpy(fx, gx, sizeof fx);
            memcpy(fy, gy, sizeof fy);
        }
        const float2 act = crowd_action(me, goal[a], q, c, fx[0], fy[0]);
        action_host[2 * a] = act.x;
        action_host[2 * a + 1] = act.y;
    }
    return RLCA_OK;
}

extern "C" int rlca_crowd_expf_host(const float *x_host, int32_t n, float *out_host)
{
    if (!x_host || !out_host || n < 0) return rlca_set_err(RLCA_ERR_INVALID, "rlca_crowd_expf_host: bad arguments");
    for (int32_t i = 0; i < n; ++i) out_host[i] = dev_expf(x_host[i]);
    return RLCA_OK;
}
