// rlca_noise.cu — sensor and actuation noise around the tick (sm_90a), C ABI in include/rlca.h, DESIGN.md §9p.
//
// rlca_noise_scan perturbs the newest frame of an observation stack in place after a tick: beam dropout and range
// noise.  rlca_noise_action turns a command into the command the robots execute: a multiplicative gain error on v and
// w.  Both are separate launches; the tick's kernels, its config and its outputs are untouched, and a run without noise
// issues neither.
//
// Every draw is a function of (seed, global agent, draw, element group, purpose | stream << 8) alone, so the noise of a
// robot is the same at any num_worlds, shard or launch shape.  Every function the kernels call is __host__ __device__
// and the file is built without FMA contraction on either side; the contract ln / sin / cos of rlca_common.cuh and
// IEEE sqrt and division make the host twins (serial loops over the same code) equal the kernels bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define NOISE_THREADS 256

struct NoiseArgs {
    float range_sigma, dropout, v_sigma, w_sigma;
    float range_max, rmax_out;            // rmax_out: the scan value of range_max, as the tick writes it
    float v_min, v_max, w_min, w_max;
    uint32_t k0, k1, stream, draw, agent0; // agent0: global index of row 0, world_offset * R
    int beams, groups;                     // groups = ceil(beams / 4)
    size_t rows;
};

// the four Philox words of (agent, draw, group, purpose) under the key
__host__ __device__ __forceinline__ void noise_words(const NoiseArgs &q, uint32_t agent, uint32_t group,
                                                     uint32_t purpose, uint32_t (&c)[4])
{
    c[0] = agent;
    c[1] = q.draw;
    c[2] = group;
    c[3] = link_word(purpose, q.stream);
    dev_philox(c, q.k0, q.k1);
}

// normals z (range noise) and uniforms u (dropout) of the four beams of group g; unused kinds are not drawn
__host__ __device__ __forceinline__ void group_draws(const NoiseArgs &q, uint32_t agent, uint32_t g, float (&z)[4],
                                                     float (&u)[4])
{
    uint32_t c[4];
    if (q.range_sigma > 0.0f) {
        noise_words(q, agent, g, PURPOSE_NOISE_RANGE, c);
        box_muller(c[0], c[1], z[0], z[1]);
        box_muller(c[2], c[3], z[2], z[3]);
    } else {
        z[0] = z[1] = z[2] = z[3] = 0.0f;
    }
    if (q.dropout > 0.0f) {
        noise_words(q, agent, g, PURPOSE_NOISE_DROPOUT, c);
#pragma unroll
        for (int j = 0; j < 4; ++j) u[j] = (float)(c[j] >> 8) * 5.9604644775390625e-08f;
    } else {
        u[0] = u[1] = u[2] = u[3] = 1.0f;       // never below a dropout of 0
    }
}

// one beam's perturbed scan value from its value o, its normal z and its uniform u
__host__ __device__ __forceinline__ float noise_beam(const NoiseArgs &q, float o, float z, float u)
{
    if (u < q.dropout) return q.rmax_out;
    if (!(q.range_sigma > 0.0f)) return o;
    const float r = (o + 0.5f) * q.range_max;
    if (!(r < q.range_max)) return o;           // no return: noise never makes one
    const float rp = fminf(fmaxf(fmaf(q.range_sigma, z, r), 0.0f), q.range_max);
    return fmaf(rp, 1.0f / 6.0f, -0.5f);
}

// clip without a comparison of two zeros, so that -0 and +0 pass unchanged on host and device alike
__host__ __device__ __forceinline__ float clip(float x, float lo, float hi)
{
    return x < lo ? lo : (x > hi ? hi : x);
}

// the executed command of one agent from its command (v, w)
__host__ __device__ __forceinline__ void noise_command(const NoiseArgs &q, uint32_t agent, float v, float w,
                                                       float &vo, float &wo)
{
    v = clip(v, q.v_min, q.v_max);
    w = clip(w, q.w_min, q.w_max);
    if (q.v_sigma > 0.0f || q.w_sigma > 0.0f) {
        uint32_t c[4];
        noise_words(q, agent, 0u, PURPOSE_NOISE_ACTION, c);
        float z1, z2;
        box_muller(c[0], c[1], z1, z2);
        v = clip(v * fmaxf(fmaf(q.v_sigma, z1, 1.0f), 0.0f), q.v_min, q.v_max);
        w = clip(w * fmaxf(fmaf(q.w_sigma, z2, 1.0f), 0.0f), q.w_min, q.w_max);
    }
    vo = v;
    wo = w;
}

// element (row, group) of the scan pass; `stack` is the row's three frames, `fresh` its was_reset flag
__host__ __device__ __forceinline__ void scan_group(const NoiseArgs &q, size_t row, int g, bool fresh, float *stack)
{
    float z[4], u[4];
    group_draws(q, q.agent0 + (uint32_t)row, (uint32_t)g, z, u);
    const int B = q.beams, b0 = 4 * g;
    float *newest = stack + 2 * (size_t)B;
    for (int j = 0; j < 4 && b0 + j < B; ++j) {
        const float v = noise_beam(q, newest[b0 + j], z[j], u[j]);
        newest[b0 + j] = v;
        if (fresh) {
            stack[b0 + j] = v;
            stack[B + b0 + j] = v;
        }
    }
}

// One thread per (row, group of four beams).  VEC: beams % 4 == 0 and a 16-byte aligned stack, 128-bit loads/stores.
template <bool VEC>
__global__ void __launch_bounds__(NOISE_THREADS) rlca_noise_scan_kernel(NoiseArgs q, const uchar4 *__restrict__ flags,
                                                                       float *__restrict__ stack)
{
    const size_t t = (size_t)blockIdx.x * NOISE_THREADS + threadIdx.x;
    if (t >= q.rows * (size_t)q.groups) return;
    const size_t row = t / (size_t)q.groups;
    const int g = (int)(t - row * (size_t)q.groups);
    const bool fresh = flags == nullptr || flags[row].w != 0;
    float *s = stack + row * 3 * (size_t)q.beams;
    if (VEC) {
        float z[4], u[4];
        group_draws(q, q.agent0 + (uint32_t)row, (uint32_t)g, z, u);
        float4 *s4 = reinterpret_cast<float4 *>(s);
        const int G = q.groups;
        float4 o = s4[2 * G + g];
        o.x = noise_beam(q, o.x, z[0], u[0]);
        o.y = noise_beam(q, o.y, z[1], u[1]);
        o.z = noise_beam(q, o.z, z[2], u[2]);
        o.w = noise_beam(q, o.w, z[3], u[3]);
        s4[2 * G + g] = o;
        if (fresh) {
            s4[g] = o;
            s4[G + g] = o;
        }
    } else {
        scan_group(q, row, g, fresh, s);
    }
}

__global__ void __launch_bounds__(NOISE_THREADS) rlca_noise_action_kernel(NoiseArgs q, const float2 *__restrict__ in,
                                                                         float2 *__restrict__ out)
{
    const size_t a = (size_t)blockIdx.x * NOISE_THREADS + threadIdx.x;
    if (a >= q.rows) return;
    const float2 c = in[a];
    float2 e;
    noise_command(q, q.agent0 + (uint32_t)a, c.x, c.y, e.x, e.y);
    out[a] = e;
}

// ------------------------------------------------------------------------------------------------ entries
static int noise_args(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw, NoiseArgs &q)
{
    if (!cfg || !p) return rlca_set_err(RLCA_ERR_INVALID, "noise: cfg or params is NULL");
    if (int rc = rlca_check_robots(cfg, "noise")) return rc;
    if (cfg->beams < 1) return rlca_set_err(RLCA_ERR_INVALID, "noise: beams must be >= 1");
    if (int rc = rlca_check_link(cfg, p->stream_id, "noise")) return rc;
    if (!finite_nonneg(p->range_sigma) || !finite_nonneg(p->v_gain_sigma) || !finite_nonneg(p->w_gain_sigma))
        return rlca_set_err(RLCA_ERR_INVALID, "noise: range_sigma, v_gain_sigma and w_gain_sigma must be finite and >= 0");
    if (!(p->dropout >= 0.0f && p->dropout <= 1.0f))
        return rlca_set_err(RLCA_ERR_INVALID, "noise: dropout must be in [0, 1]");
    q.range_sigma = p->range_sigma;
    q.dropout = p->dropout;
    q.v_sigma = p->v_gain_sigma;
    q.w_sigma = p->w_gain_sigma;
    q.range_max = cfg->range_max;
    q.rmax_out = fmaf(cfg->range_max, 1.0f / 6.0f, -0.5f);
    q.v_min = cfg->v_min;
    q.v_max = cfg->v_max;
    q.w_min = cfg->w_min;
    q.w_max = cfg->w_max;
    q.k0 = (uint32_t)p->seed;
    q.k1 = (uint32_t)(p->seed >> 32);
    q.stream = p->stream_id;
    q.draw = draw;
    q.agent0 = (uint32_t)cfg->world_offset * (uint32_t)cfg->robots_per_world;
    q.beams = cfg->beams;
    q.groups = (cfg->beams + 3) / 4;
    q.rows = (size_t)cfg->num_worlds * (size_t)cfg->robots_per_world;
    return RLCA_OK;
}

static unsigned blocks(size_t threads) { return (unsigned)((threads + NOISE_THREADS - 1) / NOISE_THREADS); }

extern "C" int rlca_noise_scan(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                               const unsigned char *flags_dev, float *stack_dev, void *stream)
{
    NoiseArgs q;
    int rc = noise_args(cfg, p, draw, q);
    if (rc) return rc;
    if (!stack_dev) return rlca_set_err(RLCA_ERR_INVALID, "rlca_noise_scan: stack_dev is NULL");
    const uchar4 *flags = reinterpret_cast<const uchar4 *>(flags_dev);
    const unsigned grid = blocks(q.rows * (size_t)q.groups);
    if ((q.beams & 3) == 0 && (reinterpret_cast<uintptr_t>(stack_dev) & 15) == 0)
        rlca_noise_scan_kernel<true><<<grid, NOISE_THREADS, 0, (cudaStream_t)stream>>>(q, flags, stack_dev);
    else
        rlca_noise_scan_kernel<false><<<grid, NOISE_THREADS, 0, (cudaStream_t)stream>>>(q, flags, stack_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_noise_action(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                                 const float *action_in_dev, float *action_out_dev, void *stream)
{
    NoiseArgs q;
    int rc = noise_args(cfg, p, draw, q);
    if (rc) return rc;
    if (!action_in_dev || !action_out_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_noise_action: action_in_dev or action_out_dev is NULL");
    rlca_noise_action_kernel<<<blocks(q.rows), NOISE_THREADS, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const float2 *>(action_in_dev), reinterpret_cast<float2 *>(action_out_dev));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_noise_scan_host(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                                    const unsigned char *flags_host, float *stack_host)
{
    NoiseArgs q;
    int rc = noise_args(cfg, p, draw, q);
    if (rc) return rc;
    if (!stack_host) return rlca_set_err(RLCA_ERR_INVALID, "rlca_noise_scan_host: stack_host is NULL");
    for (size_t row = 0; row < q.rows; ++row) {
        const bool fresh = flags_host == nullptr || flags_host[4 * row + 3] != 0;
        for (int g = 0; g < q.groups; ++g) scan_group(q, row, g, fresh, stack_host + row * 3 * (size_t)q.beams);
    }
    return RLCA_OK;
}

extern "C" int rlca_noise_action_host(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                                      const float *action_in_host, float *action_out_host)
{
    NoiseArgs q;
    int rc = noise_args(cfg, p, draw, q);
    if (rc) return rc;
    if (!action_in_host || !action_out_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_noise_action_host: action_in_host or action_out_host is NULL");
    for (size_t a = 0; a < q.rows; ++a)
        noise_command(q, q.agent0 + (uint32_t)a, action_in_host[2 * a], action_in_host[2 * a + 1],
                      action_out_host[2 * a], action_out_host[2 * a + 1]);
    return RLCA_OK;
}
