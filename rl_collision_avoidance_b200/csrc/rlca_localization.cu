// rlca_localization.cu — localization error in the policy's goal and speed inputs (sm_90a), C ABI in include/rlca.h,
// DESIGN.md §9s.
//
// rlca_localization_observe turns the local goal and speed the tick wrote into what a robot with a localizer and
// odometry reads: the local goal from a believed pose (x + ex, y + ey, theta + etheta) and the speed with white noise.
// The pose error e follows a first-order Gauss-Markov process per agent and component, whose standard deviations are
// drawn when the agent starts an episode.  It is a separate launch after the tick; the tick's kernels, its config and
// its outputs are untouched, and a run without localization error issues none.
//
// The error and its standard deviations are state across ticks, so this is a file of its own, as latency and dynamics
// are.  Every draw is a function of (seed, global agent, draw, group, 0xE7 | stream << 8) alone; the local goal is the
// tick's own goal_speed and dev_sincosf, Box-Muller is noise's, and the file is built without FMA contraction on either
// side, so the host twin (a serial loop over the same code) equals the kernel bit for bit at any num_worlds, shard or
// launch shape.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define LOCALIZATION_THREADS 256
#define PURPOSE_POSE_ERROR 0xE7u

struct LocalizationArgs {
    float xy_lo, xy_span, th_lo, th_span;       // sigma = lo + span u
    float rho, kappa;                           // e <- rho e + kappa sigma xi
    float v_sigma, w_sigma;
    uint32_t k0, k1, stream, draw, agent0;      // agent0: global index of row 0, world_offset * R
    size_t rows;
};

// one step of a component's Gauss-Markov error: n = sigma xi is a draw of the stationary distribution, which a fresh
// row takes as it is; rho = 1 (kappa = 0, a constant offset) holds e as it is, so its bits never change in an episode
__host__ __device__ __forceinline__ float gauss_markov(const LocalizationArgs &q, bool fresh, float e, float n)
{
    return fresh ? n : (q.kappa == 0.0f ? e : q.rho * e + q.kappa * n);
}

// the believed goal and speed of row a from its pose, goal and true goal / speed: a fresh row draws its standard
// deviations and starts from the stationary distribution; a component whose error is exactly 0 keeps the true value
__host__ __device__ __forceinline__ float4 localization_agent(const LocalizationArgs &q, size_t a, bool fresh,
                                                              float4 pose, float4 goal, float4 gs, float4 *err,
                                                              float2 *sigma)
{
    const uint32_t agent = q.agent0 + (uint32_t)a, purpose = PURPOSE_POSE_ERROR | (q.stream << 8);
    uint32_t c0[4] = {agent, q.draw, 0u, purpose}, c1[4] = {agent, q.draw, 1u, purpose};
    dev_philox(c0, q.k0, q.k1);
    dev_philox(c1, q.k0, q.k1);
    float zx, zy, zt, zv, zw, unused;
    box_muller(c0[0], c0[1], zx, zy);
    box_muller(c0[2], c0[3], zt, zv);
    box_muller(c1[0], c1[1], zw, unused);
    float2 sg;
    if (fresh) {
        sg.x = q.xy_lo + q.xy_span * ((float)(c1[2] >> 8) * 5.9604644775390625e-08f);
        sg.y = q.th_lo + q.th_span * ((float)(c1[3] >> 8) * 5.9604644775390625e-08f);
        sigma[a] = sg;
    } else {
        sg = sigma[a];
    }
    float4 e = fresh ? make_float4(0.0f, 0.0f, 0.0f, 0.0f) : err[a];
    e.x = gauss_markov(q, fresh, e.x, sg.x * zx);
    e.y = gauss_markov(q, fresh, e.y, sg.x * zy);
    e.z = gauss_markov(q, fresh, e.z, sg.y * zt);
    err[a] = e;
    float4 bp = pose;
    if (e.x != 0.0f) bp.x = pose.x + e.x;
    if (e.y != 0.0f) bp.y = pose.y + e.y;
    if (e.z != 0.0f) bp.z = pose.z + e.z;
    float s, c;
    dev_sincosf(bp.z, s, c);
    float4 out = goal_speed(bp, goal, s, c);
    out.z = q.v_sigma > 0.0f ? gs.z + q.v_sigma * zv : gs.z;
    out.w = q.w_sigma > 0.0f ? gs.w + q.w_sigma * zw : gs.w;
    return out;
}

// One thread per agent.  gs_in and gs_out may be the same buffer: each thread reads its row before it writes it.
__global__ void __launch_bounds__(LOCALIZATION_THREADS)
    rlca_localization_kernel(LocalizationArgs q, const uchar4 *__restrict__ flags, const float4 *__restrict__ pose,
                             const float4 *__restrict__ goal, const float4 *gs_in, float4 *gs_out,
                             float4 *__restrict__ err, float2 *__restrict__ sigma)
{
    const size_t a = (size_t)blockIdx.x * LOCALIZATION_THREADS + threadIdx.x;
    if (a >= q.rows) return;
    const bool fresh = flags == nullptr || flags[a].w != 0;
    const float4 g = gs_in[a];
    gs_out[a] = localization_agent(q, a, fresh, pose[a], goal[a], g, err, sigma);
}

// ------------------------------------------------------------------------------------------------ entries
static bool finite_nonneg(float v) { return v >= 0.0f && v < INFINITY; }

static int localization_args(const rlca_env_config *cfg, const rlca_localization_params *p,
                             const rlca_localization_state *st, uint32_t draw, const rlca_env_state *env,
                             const float *gs_in, const float *gs_out, LocalizationArgs &q)
{
    if (!cfg || !p || !st || !env) return rlca_set_err(RLCA_ERR_INVALID, "localization: cfg, params, state or env state is NULL");
    if (!st->err || !st->sigma) return rlca_set_err(RLCA_ERR_INVALID, "localization: state err or sigma is NULL");
    if (!env->pose_dev || !env->goal_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "localization: env state pose or goal is NULL");
    if (!gs_in || !gs_out) return rlca_set_err(RLCA_ERR_INVALID, "localization: gs_in or gs_out is NULL");
    if (cfg->robots_per_world < 1 || cfg->robots_per_world > RLCA_MAX_ROBOTS_PER_WORLD || cfg->num_worlds < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "localization: robots_per_world must be in 1..64 and num_worlds >= 1");
    if (cfg->world_offset < 0) return rlca_set_err(RLCA_ERR_INVALID, "localization: world_offset must be >= 0");
    if (!finite_nonneg(p->xy_lo) || !finite_nonneg(p->xy_hi) || !(p->xy_lo <= p->xy_hi) ||
        !finite_nonneg(p->theta_lo) || !finite_nonneg(p->theta_hi) || !(p->theta_lo <= p->theta_hi))
        return rlca_set_err(RLCA_ERR_INVALID, "localization: every sigma range must be finite with 0 <= lo <= hi");
    if (!finite_nonneg(p->v_sigma) || !finite_nonneg(p->w_sigma))
        return rlca_set_err(RLCA_ERR_INVALID, "localization: v_sigma and w_sigma must be finite and >= 0");
    if (!(p->tau >= 0.0f)) return rlca_set_err(RLCA_ERR_INVALID, "localization: tau must be >= 0 or +inf");
    if (p->stream_id >= (1u << 24)) return rlca_set_err(RLCA_ERR_INVALID, "localization: stream_id must be below 2^24");
    // rho = exp(-dt / tau) and kappa = sqrt(1 - rho^2), once here in double: the kernel and the twin share the floats
    double rho = 0.0, kappa = 1.0;
    if (p->tau == INFINITY) {
        rho = 1.0;
        kappa = 0.0;
    } else if (p->tau > 0.0f) {
        rho = exp(-(double)cfg->dt / (double)p->tau);
        kappa = sqrt(1.0 - rho * rho);
    }
    q.xy_lo = p->xy_lo;
    q.xy_span = p->xy_hi - p->xy_lo;
    q.th_lo = p->theta_lo;
    q.th_span = p->theta_hi - p->theta_lo;
    q.rho = (float)rho;
    q.kappa = (float)kappa;
    q.v_sigma = p->v_sigma;
    q.w_sigma = p->w_sigma;
    q.k0 = (uint32_t)p->seed;
    q.k1 = (uint32_t)(p->seed >> 32);
    q.stream = p->stream_id;
    q.draw = draw;
    q.agent0 = (uint32_t)cfg->world_offset * (uint32_t)cfg->robots_per_world;
    q.rows = (size_t)cfg->num_worlds * (size_t)cfg->robots_per_world;
    return RLCA_OK;
}

extern "C" int rlca_localization_observe(const rlca_env_config *cfg, const rlca_localization_params *p,
                                         const rlca_localization_state *state, uint32_t draw,
                                         const unsigned char *flags_dev, const rlca_env_state *state_env,
                                         const float *gs_in_dev, float *gs_out_dev, void *stream)
{
    LocalizationArgs q;
    int rc = localization_args(cfg, p, state, draw, state_env, gs_in_dev, gs_out_dev, q);
    if (rc) return rc;
    const unsigned grid = (unsigned)((q.rows + LOCALIZATION_THREADS - 1) / LOCALIZATION_THREADS);
    rlca_localization_kernel<<<grid, LOCALIZATION_THREADS, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const uchar4 *>(flags_dev), reinterpret_cast<const float4 *>(state_env->pose_dev),
        reinterpret_cast<const float4 *>(state_env->goal_dev), reinterpret_cast<const float4 *>(gs_in_dev),
        reinterpret_cast<float4 *>(gs_out_dev), reinterpret_cast<float4 *>(state->err),
        reinterpret_cast<float2 *>(state->sigma));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_localization_observe_host(const rlca_env_config *cfg, const rlca_localization_params *p,
                                              const rlca_localization_state *state, uint32_t draw,
                                              const unsigned char *flags_host, const rlca_env_state *state_host,
                                              const float *gs_in_host, float *gs_out_host)
{
    LocalizationArgs q;
    int rc = localization_args(cfg, p, state, draw, state_host, gs_in_host, gs_out_host, q);
    if (rc) return rc;
    const float4 *pose = reinterpret_cast<const float4 *>(state_host->pose_dev);
    const float4 *goal = reinterpret_cast<const float4 *>(state_host->goal_dev);
    float4 *err = reinterpret_cast<float4 *>(state->err);
    float2 *sigma = reinterpret_cast<float2 *>(state->sigma);
    for (size_t a = 0; a < q.rows; ++a) {
        const bool fresh = flags_host == nullptr || flags_host[4 * a + 3] != 0;
        const float4 g = make_float4(gs_in_host[4 * a], gs_in_host[4 * a + 1], gs_in_host[4 * a + 2],
                                     gs_in_host[4 * a + 3]);
        const float4 o = localization_agent(q, a, fresh, pose[a], goal[a], g, err, sigma);
        gs_out_host[4 * a] = o.x;
        gs_out_host[4 * a + 1] = o.y;
        gs_out_host[4 * a + 2] = o.z;
        gs_out_host[4 * a + 3] = o.w;
    }
    return RLCA_OK;
}
