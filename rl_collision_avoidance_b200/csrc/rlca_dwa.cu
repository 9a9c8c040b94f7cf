// rlca_dwa.cu — the dynamic-window baseline (sm_90a), C ABI in include/rlca.h, DESIGN.md §9u.
//
// rlca_dwa_action drives every robot from what the policy reads: the newest frame of its scan stack, its local goal and
// its speed (gs).  Per robot (Fox, Burgard, Thrun 1997) a v_samples x w_samples grid of constant-(v, w) commands over
// the dynamic window is scored against every scan return within reach: the arc length a disc of radius rho drives
// before it first touches a return (closed form, below), admissibility by the braking distance, and a score of goal
// heading, clearance and speed.  The best admissible candidate is the command; with none, (0, 0) and status 1.
//
// One warp per robot, 8 robots per CTA.  The warp loads frame 2 coalesced and compacts the returns within reach into
// per-warp shared memory in beam order (ballot + popc); lanes take candidates lane, lane + 32, ... and loop over the
// shared points (every lane reads the same point: a broadcast); a (score, index) warp argmax finishes the robot.  Each
// candidate walks the points in beam order on both entries, the argmax with its lowest-index tie-break does not depend
// on the order of the reduction, every per-point and per-candidate function is shared with the host twin, and the file
// is built without FMA contraction on either side, so the host twin (a serial loop over the same code) equals the
// kernel bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define DWA_WARPS 8
#define DWA_THREADS (DWA_WARPS * 32)
#define DWA_PI 3.14159265358979324f
#define DWA_TWO_PI 6.28318530717958648f

struct DwaArgs {
    int nv, nw, ncand, beams;
    float rho, rho2, horizon, heading_time;
    float adt, aadt;                            // window half-widths accel dt, angular_accel dt; 0 = the whole box
    float brake2;                               // 2 brake
    float hw, cw, sw, cap;
    float dt, range_max, v_min, v_max, w_min, w_max;
    size_t rows;
};

struct DwaWindow {
    float v_lo, v_hi, w_lo, w_hi;
};

// the window around the robot's speed (v0, w0), itself clamped into the action box first (a believed speed under
// localization error may lie outside it), so the window is never empty
__host__ __device__ __forceinline__ DwaWindow dwa_window(const DwaArgs &q, float v0, float w0)
{
    DwaWindow d;
    v0 = fminf(fmaxf(v0, q.v_min), q.v_max);
    w0 = fminf(fmaxf(w0, q.w_min), q.w_max);
    d.v_lo = q.adt > 0.0f ? fmaxf(q.v_min, v0 - q.adt) : q.v_min;
    d.v_hi = q.adt > 0.0f ? fminf(q.v_max, v0 + q.adt) : q.v_max;
    d.w_lo = q.aadt > 0.0f ? fmaxf(q.w_min, w0 - q.aadt) : q.w_min;
    d.w_hi = q.aadt > 0.0f ? fminf(q.w_max, w0 + q.aadt) : q.w_max;
    return d;
}

// sample i of n over [lo, hi]: both ends exactly, the midpoint when n = 1
__host__ __device__ __forceinline__ float dwa_sample(float lo, float hi, int i, int n)
{
    if (n == 1) return 0.5f * (lo + hi);
    if (i == n - 1) return hi;
    return lo + (hi - lo) * ((float)i / (float)(n - 1));
}

// a return at range r (scan value s) of beam direction cs: a point in the robot frame when it lies within reach
__host__ __device__ __forceinline__ bool dwa_point(const DwaArgs &q, float s, float2 cs, float reach, float2 &pt,
                                                   bool &touch)
{
    const float r = (s + 0.5f) * q.range_max;
    const bool ret = r < q.range_max;
    touch = ret && r < q.rho;
    pt = make_float2(r * cs.x, r * cs.y);
    return ret && r <= reach;
}

// Arc length the disc drives on the candidate's path before it first touches the point (px, py), +inf if it never
// does.  The point lies at least rho from the robot (a return within rho is caught before, as touch).
//   straight: x - sqrt(rho^2 - y^2) for |y| < rho ahead.
//   arc of radius R = v / |w| about C = (0, +-R) (y mirrored for w < 0, so C = (0, R) and the motion is
//   counter-clockwise): with q = D^2 - R^2 = x^2 + y^2 - 2 y R (D = |P - C|), the path's disc meets the point iff
//   |D - R| < rho, i.e. |q - rho^2| < 2 R rho.  The contact lies at the angle alpha before the point's own angle theta_P
//   (swept from the robot, in [0, 2 pi)), alpha from the law of cosines in the triangle (C, P, contact centre):
//   2 R D cos(alpha) = 2 R^2 + q - rho^2, 2 R D sin(alpha) = sqrt((rho^2 - (D - R)^2) ((D + R)^2 - rho^2)), with
//   D - R = q / (D + R).  Contact arc length R (theta_P - alpha).
__host__ __device__ __forceinline__ float dwa_contact(const DwaArgs &q, bool straight, bool mirror, float R, float two_r_rho,
                                                      float2 p, float r2)
{
    if (straight) {
        if (p.x > 0.0f && fabsf(p.y) < q.rho) return fmaxf(p.x - sqrtf(q.rho2 - p.y * p.y), 0.0f);
        return INFINITY;
    }
    const float y = mirror ? -p.y : p.y;
    const float qq = r2 - 2.0f * y * R;
    if (!(fabsf(qq - q.rho2) < two_r_rho)) return INFINITY;
    const float D = sqrtf(fmaxf(R * R + qq, 0.0f));
    const float dm = qq / (D + R);
    const float e1 = fmaxf(q.rho2 - dm * dm, 0.0f);
    const float sp = D + R;
    const float e2 = fmaxf(sp * sp - q.rho2, 0.0f);
    const float alpha = dev_atan2f(sqrtf(e1 * e2), 2.0f * R * R + qq - q.rho2);
    float th = dev_atan2f(p.x, R - y);
    if (th < 0.0f) th += DWA_TWO_PI;
    return R * fmaxf(th - alpha, 0.0f);
}

// |w| below this drives straight: a radius v / |w| beyond 1e6 m is a line, and its square would overflow
#define DWA_STRAIGHT_W 1e-6f

// candidate c of the window: its command, clearance over the n points, admissibility and score
__host__ __device__ __forceinline__ float dwa_candidate(const DwaArgs &q, const DwaWindow &win, float gx, float gy,
                                                        const float2 *pts, int n, bool touch, int c, float &v, float &w,
                                                        float &clear, bool &admissible)
{
    v = dwa_sample(win.v_lo, win.v_hi, c / q.nw, q.nv);
    w = dwa_sample(win.w_lo, win.w_hi, c % q.nw, q.nw);
    const bool straight = fabsf(w) < DWA_STRAIGHT_W;
    float cl;
    if (touch) {
        cl = 0.0f;
    } else if (v == 0.0f) {
        cl = q.cap;
    } else {
        const bool mirror = w < 0.0f;
        const float R = straight ? 0.0f : v / fabsf(w);
        const float two_r_rho = 2.0f * R * q.rho;
        // A point at range r is touched no earlier than r - rho along any path, so one with r >= cl + rho cannot lower
        // the clearance and is skipped.  Both entries walk the points in beam order, so they skip the same ones.
        cl = v * q.horizon;
        float lim = (cl + q.rho) * (cl + q.rho);
        for (int i = 0; i < n; ++i) {
            const float2 p = pts[i];
            const float r2 = p.x * p.x + p.y * p.y;
            if (r2 >= lim) continue;
            const float c = dwa_contact(q, straight, mirror, R, two_r_rho, p, r2);
            if (c < cl) {
                cl = c;
                lim = (cl + q.rho) * (cl + q.rho);
            }
        }
    }
    clear = cl;
    admissible = cl > 0.0f && cl >= v * q.dt + v * v / q.brake2;
    // the pose after heading_time on the candidate's arc, and the goal's bearing from it
    float hx, hy, th;
    if (v == 0.0f) {
        hx = 0.0f;
        hy = 0.0f;
        th = w * q.heading_time;
    } else if (straight) {
        hx = v * q.heading_time;
        hy = 0.0f;
        th = 0.0f;
    } else {
        th = w * q.heading_time;
    }
    float s, co;
    dev_sincosf(th, s, co);
    if (v != 0.0f && !straight) {
        const float Rs = v / w;
        hx = Rs * s;
        hy = co > -0.5f ? hx * (s / (1.0f + co)) : Rs * (1.0f - co);      // R (1 - cos) without the cancellation
    }
    const float dx = gx - hx, dy = gy - hy;
    const float bearing = dev_atan2f(dy * co - dx * s, dx * co + dy * s);
    return q.hw * (1.0f - fabsf(bearing) / DWA_PI) + q.cw * (fminf(cl, q.cap) / q.cap) + q.sw * (v / q.v_max);
}

__global__ void __launch_bounds__(DWA_THREADS)
    rlca_dwa_kernel(DwaArgs q, const float2 *__restrict__ cs, const float *__restrict__ stack,
                    const float4 *__restrict__ gs, float2 *__restrict__ action, int32_t *__restrict__ status)
{
    __shared__ float2 pts[DWA_WARPS][RLCA_DWA_MAX_BEAMS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t a = (size_t)blockIdx.x * DWA_WARPS + warp;
    if (a >= q.rows) return;
    const float4 g = gs[a];
    const DwaWindow win = dwa_window(q, g.z, g.w);
    const float reach = win.v_hi * q.horizon + q.rho;
    const float *scan = stack + (a * 3 + 2) * (size_t)q.beams;
    float2 *mine = pts[warp];
    int n = 0;
    bool touch = false;
    for (int b0 = 0; b0 < q.beams; b0 += 32) {
        const int j = b0 + lane;
        float2 pt = make_float2(0.0f, 0.0f);
        bool t = false, hit = false;
        if (j < q.beams) hit = dwa_point(q, scan[j], cs[j], reach, pt, t);
        touch |= t;
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (hit) mine[n + __popc(m & ((1u << lane) - 1u))] = pt;
        n += __popc(m);
    }
    touch = __any_sync(0xffffffffu, touch);
    __syncwarp();
    float best = -INFINITY;
    int bi = q.ncand;
    for (int c = lane; c < q.ncand; c += 32) {
        float v, w, cl;
        bool adm;
        const float sc = dwa_candidate(q, win, g.x, g.y, mine, n, touch, c, v, w, cl, adm);
        if (adm && sc > best) {
            best = sc;
            bi = c;
        }
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        const float os = __shfl_xor_sync(0xffffffffu, best, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (os > best || (os == best && oi < bi)) {
            best = os;
            bi = oi;
        }
    }
    if (lane == 0) {
        const bool ok = bi < q.ncand;
        action[a] = ok ? make_float2(dwa_sample(win.v_lo, win.v_hi, bi / q.nw, q.nv),
                                     dwa_sample(win.w_lo, win.w_hi, bi % q.nw, q.nw))
                       : make_float2(0.0f, 0.0f);
        status[a] = ok ? 0 : 1;
    }
}

// ------------------------------------------------------------------------------------------------ entries
static bool finite_pos(float v) { return v > 0.0f && v < INFINITY; }

static int dwa_args(const rlca_env_config *cfg, const rlca_dwa_params *p, const void *cs, const void *stack,
                    const void *gs, const void *action, const void *status, DwaArgs &q)
{
    if (!cfg || !p) return rlca_set_err(RLCA_ERR_INVALID, "dwa: cfg or params is NULL");
    if (!cs || !stack || !gs || !action || !status)
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: beam table, stack, gs, action or status is NULL");
    if (cfg->robots_per_world < 1 || cfg->num_worlds < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: robots_per_world and num_worlds must be >= 1");
    if (cfg->beams < 2 || cfg->beams > RLCA_DWA_MAX_BEAMS)
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: beams must be in 2..512");
    if (!finite_pos(cfg->range_max) || !finite_pos(cfg->dt) || !finite_pos(cfg->v_max) ||
        !(cfg->v_min <= cfg->v_max) || !(cfg->w_min <= cfg->w_max) || !(fabsf(cfg->v_min) < INFINITY) ||
        !(fabsf(cfg->w_min) < INFINITY) || !(fabsf(cfg->w_max) < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: the config needs finite range_max, dt, v_max > 0 and an action box");
    if (p->v_samples < 1 || p->w_samples < 1 ||
        (int64_t)p->v_samples * (int64_t)p->w_samples > RLCA_DWA_MAX_CANDIDATES)
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: v_samples and w_samples must be >= 1 with a product of at most 1024");
    if (!finite_pos(p->radius) || !finite_pos(p->horizon) || !finite_pos(p->brake) || !finite_pos(p->clearance_cap))
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: radius, horizon, brake and clearance_cap must be finite and > 0");
    if (!finite_nonneg(p->heading_time) || !finite_nonneg(p->accel) || !finite_nonneg(p->angular_accel))
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: heading_time, accel and angular_accel must be finite and >= 0");
    if (!finite_nonneg(p->heading_weight) || !finite_nonneg(p->clearance_weight) || !finite_nonneg(p->speed_weight))
        return rlca_set_err(RLCA_ERR_INVALID, "dwa: the weights must be finite and >= 0");
    q.nv = p->v_samples;
    q.nw = p->w_samples;
    q.ncand = p->v_samples * p->w_samples;
    q.beams = cfg->beams;
    q.rho = p->radius;
    q.rho2 = p->radius * p->radius;
    q.horizon = p->horizon;
    q.heading_time = p->heading_time;
    q.adt = p->accel * cfg->dt;
    q.aadt = p->angular_accel * cfg->dt;
    q.brake2 = 2.0f * p->brake;
    q.hw = p->heading_weight;
    q.cw = p->clearance_weight;
    q.sw = p->speed_weight;
    q.cap = p->clearance_cap;
    q.dt = cfg->dt;
    q.range_max = cfg->range_max;
    q.v_min = cfg->v_min;
    q.v_max = cfg->v_max;
    q.w_min = cfg->w_min;
    q.w_max = cfg->w_max;
    q.rows = (size_t)cfg->num_worlds * (size_t)cfg->robots_per_world;
    return RLCA_OK;
}

extern "C" int rlca_dwa_action(const rlca_env_config *cfg, const rlca_dwa_params *p, const float *beam_cos_sin_dev,
                               const float *stack_dev, const float *gs_dev, float *action_dev, int32_t *status_dev,
                               void *stream)
{
    DwaArgs q;
    int rc = dwa_args(cfg, p, beam_cos_sin_dev, stack_dev, gs_dev, action_dev, status_dev, q);
    if (rc) return rc;
    const unsigned grid = (unsigned)((q.rows + DWA_WARPS - 1) / DWA_WARPS);
    rlca_dwa_kernel<<<grid, DWA_THREADS, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const float2 *>(beam_cos_sin_dev), stack_dev, reinterpret_cast<const float4 *>(gs_dev),
        reinterpret_cast<float2 *>(action_dev), status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_dwa_action_host(const rlca_env_config *cfg, const rlca_dwa_params *p, const float *beam_cos_sin_host,
                                    const float *stack_host, const float *gs_host, float *action_host,
                                    int32_t *status_host, float *clearance_host, float *score_host)
{
    DwaArgs q;
    int rc = dwa_args(cfg, p, beam_cos_sin_host, stack_host, gs_host, action_host, status_host, q);
    if (rc) return rc;
    const float2 *cs = reinterpret_cast<const float2 *>(beam_cos_sin_host);
    float2 pts[RLCA_DWA_MAX_BEAMS];
    for (size_t a = 0; a < q.rows; ++a) {
        const float *g = gs_host + 4 * a;
        const DwaWindow win = dwa_window(q, g[2], g[3]);
        const float reach = win.v_hi * q.horizon + q.rho;
        const float *scan = stack_host + (a * 3 + 2) * (size_t)q.beams;
        int n = 0;
        bool touch = false;
        for (int j = 0; j < q.beams; ++j) {
            float2 pt;
            bool t;
            if (dwa_point(q, scan[j], cs[j], reach, pt, t)) pts[n++] = pt;
            touch |= t;
        }
        float best = -INFINITY, bv = 0.0f, bw = 0.0f;
        bool found = false;
        for (int c = 0; c < q.ncand; ++c) {
            float v, w, cl;
            bool adm;
            const float sc = dwa_candidate(q, win, g[0], g[1], pts, n, touch, c, v, w, cl, adm);
            if (clearance_host) clearance_host[a * q.ncand + c] = cl;
            if (score_host) score_host[a * q.ncand + c] = sc;
            if (adm && sc > best) {
                best = sc;
                bv = v;
                bw = w;
                found = true;
            }
        }
        action_host[2 * a] = found ? bv : 0.0f;
        action_host[2 * a + 1] = found ? bw : 0.0f;
        status_host[a] = found ? 0 : 1;
    }
    return RLCA_OK;
}
