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
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define ORCA_THREADS 256
#define ORCA_WARPS (ORCA_THREADS / 32)
#define ORCA_MAX_LINES (RLCA_MAX_ROBOTS_PER_WORLD - 1)
#define NH_ORCA_VERTS RLCA_NH_ORCA_VERTS
#define NH_MAX_LINES (NH_ORCA_VERTS + ORCA_MAX_LINES)
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

// NH = false: ORCA-DD (h unused); NH = true: NH-ORCA, P's lines first in the list.
template <bool NH>
__global__ void __launch_bounds__(ORCA_THREADS) rlca_orca_kernel(int n, int R, OrcaParams q, NhParams h,
                                                                  const float4 *__restrict__ pose,
                                                                  const float4 *__restrict__ goal,
                                                                  const int4 *__restrict__ meta,
                                                                  float2 *__restrict__ action,
                                                                  float2 *__restrict__ velocity,
                                                                  int32_t *__restrict__ status)
{
    constexpr int max_lines = NH ? NH_MAX_LINES : ORCA_MAX_LINES;
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
    if (fail < nl) lp3_warp(lines, nl, fail, NH ? h.nv : 0, q.v_max, s_proj[warp], rx, ry, lane);
    if (lane == 0) {
        action[a] = NH ? nh_track(me, rx, ry, q, h) : orca_track(me, rx, ry, q);
        if (velocity) velocity[a] = make_float2(rx, ry);
        if (status) status[a] = fail < nl;
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
    OrcaLine proj[NH_MAX_LINES];
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
    rlca_orca_kernel<false><<<(n + ORCA_WARPS - 1) / ORCA_WARPS, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
        n, cfg->robots_per_world, q, none, reinterpret_cast<const float4 *>(state->pose_dev),
        reinterpret_cast<const float4 *>(state->goal_dev), reinterpret_cast<const int4 *>(state->meta_dev),
        reinterpret_cast<float2 *>(action_dev), reinterpret_cast<float2 *>(velocity_dev), status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

// The per-agent steps of rlca_orca_kernel<NH> by serial loops; h = NULL is ORCA-DD.
static void host_actions(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                         const int32_t *meta_host, const OrcaParams &q, const NhParams *h, float *action_host,
                         float *velocity_host, int32_t *status_host)
{
    const float4 *pose = reinterpret_cast<const float4 *>(pose_host), *goal = reinterpret_cast<const float4 *>(goal_host);
    const int4 *meta = reinterpret_cast<const int4 *>(meta_host);
    const int R = cfg->robots_per_world, n = R * cfg->num_worlds, hard = h ? h->nv : 0;
    OrcaLine lines[NH_MAX_LINES];
    for (int a = 0; a < n; ++a) {
        const int base = a - a % R;
        const OrcaAgent me = orca_agent(pose, goal, meta, a);
        int nl = 0;
        for (; nl < hard; ++nl) lines[nl] = nh_hard_line(me, h->edge[nl]);
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
        if (status_host) status_host[a] = fail < nl;
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
    host_actions(cfg, pose_host, goal_host, meta_host, q, nullptr, action_host, velocity_host, status_host);
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
    rlca_orca_kernel<true><<<(n + ORCA_WARPS - 1) / ORCA_WARPS, ORCA_THREADS, 0, (cudaStream_t)stream>>>(
        n, cfg->robots_per_world, q, h, reinterpret_cast<const float4 *>(state->pose_dev),
        reinterpret_cast<const float4 *>(state->goal_dev), reinterpret_cast<const int4 *>(state->meta_dev),
        reinterpret_cast<float2 *>(action_dev), reinterpret_cast<float2 *>(velocity_dev), status_dev);
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
    host_actions(cfg, pose_host, goal_host, meta_host, q, &h, action_host, velocity_host, status_host);
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
