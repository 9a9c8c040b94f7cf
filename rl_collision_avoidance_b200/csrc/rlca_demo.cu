// rlca_demo.cu — demonstration recording on the device (sm_90a), C ABI in include/rlca.h, DESIGN.md §9g.
//
// rlca_demo_append runs before each rlca_env_step and appends one row (scan stack, local goal | speed, clipped action)
// per recorded agent to a fixed-capacity dataset.  Rows are ordered by agent index within a call; the row of an agent
// is the number of recorded agents before it, which every CTA counts itself over the agents ahead of its own
// (__syncthreads_count, no atomics), so the order and the contents do not depend on the schedule.  The count of rows
// held stays on the device: the last CTA to finish (a completion ticket, the one atomic) writes it.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define DEMO_THREADS 256
#define DEMO_AGENTS 8          // agents per CTA: 8 stacks of 384 float4 = 12 float4 per thread at 512 beams

// The recording rule: the agent's action on this tick comes from the caller and drives an episode that has not ended.
//   auto_reset 1: always (a done agent re-spawns inside the tick);
//   auto_reset 2: not latched (meta.w == 0): the tick idles a latched agent on its last command;
//   auto_reset 0: not done on the previous tick (flags NULL = none was): the caller stops such an agent.
__device__ __forceinline__ int demo_recorded(int auto_reset, const int4 *__restrict__ meta,
                                             const uint8_t *__restrict__ flags, int i)
{
    if (auto_reset == 2) return meta[i].w == 0;
    if (auto_reset == 0) return flags == nullptr || flags[4 * i] == 0;
    return 1;
}

__global__ void __launch_bounds__(DEMO_THREADS)
demo_append_kernel(int n, int auto_reset, int row4, float v_min, float v_max, float w_min, float w_max,
                   const float4 *__restrict__ stack, const float4 *__restrict__ gs, const float2 *__restrict__ action,
                   const int4 *__restrict__ meta, const uint8_t *__restrict__ flags, float4 *__restrict__ obs_out,
                   float4 *__restrict__ gs_out, float2 *__restrict__ act_out, unsigned long long *count,
                   long long capacity)
{
    __shared__ int rank[DEMO_AGENTS];       // row of each of this CTA's agents after `base`, -1 = not recorded
    __shared__ long long base;
    __shared__ int last;
    const int a0 = blockIdx.x * DEMO_AGENTS;
    if (threadIdx.x == 0) base = (long long)__ldcg(count);      // read before this CTA takes its ticket
    int before = 0;
    for (int j0 = 0; j0 < a0; j0 += DEMO_THREADS) {
        const int j = j0 + threadIdx.x;
        before += __syncthreads_count(j < a0 && demo_recorded(auto_reset, meta, flags, j));
    }
    if (threadIdx.x == 0) {
        int r = before;
        for (int k = 0; k < DEMO_AGENTS; ++k) {
            const int i = a0 + k;
            rank[k] = (i < n && demo_recorded(auto_reset, meta, flags, i)) ? r++ : -1;
        }
    }
    __syncthreads();
    const long long b = base;
    if (b < capacity) {
        for (int t = threadIdx.x; t < DEMO_AGENTS * row4; t += DEMO_THREADS) {
            const int k = t / row4, c = t - k * row4;
            const long long row = b + rank[k];
            if (rank[k] >= 0 && row < capacity) obs_out[row * row4 + c] = stack[(size_t)(a0 + k) * row4 + c];
        }
        if (threadIdx.x < DEMO_AGENTS) {
            const int k = threadIdx.x, i = a0 + k;
            const long long row = b + rank[k];
            if (rank[k] >= 0 && row < capacity) {
                gs_out[row] = gs[i];
                // the clip of rlca_physics_kernel, non-finite (and |x| > 3e38) -> 0 included
                float v = action[i].x, w = action[i].y;
                if (!(fabsf(v) <= 3.0e38f)) v = 0.0f;
                if (!(fabsf(w) <= 3.0e38f)) w = 0.0f;
                act_out[row] = make_float2(fminf(fmaxf(v, v_min), v_max), fminf(fmaxf(w, w_min), w_max));
            }
        }
    }
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(count + 1, 1ull) == (unsigned long long)(gridDim.x - 1);
    }
    __syncthreads();
    if (last) {                               // every CTA has read the old count: the new one can be written
        int total = 0;
        for (int j0 = 0; j0 < n; j0 += DEMO_THREADS) {
            const int j = j0 + threadIdx.x;
            total += __syncthreads_count(j < n && demo_recorded(auto_reset, meta, flags, j));
        }
        if (threadIdx.x == 0) {
            count[0] = (unsigned long long)min(capacity, b + total);
            count[1] = 0ull;
        }
    }
}

extern "C" int rlca_demo_append(const rlca_env_config *cfg, const rlca_env_state *state, const rlca_step_io *io,
                                const rlca_demo_set *demo, void *stream)
{
    if (!cfg || !state || !io || !demo) return rlca_set_err(RLCA_ERR_INVALID, "rlca_demo_append: NULL argument");
    if (cfg->robots_per_world < 1 || cfg->robots_per_world > RLCA_MAX_ROBOTS_PER_WORLD || cfg->num_worlds < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "cfg has no robots");
    if (cfg->auto_reset < 0 || cfg->auto_reset > 2) return rlca_set_err(RLCA_ERR_INVALID, "cfg.auto_reset must be 0, 1 or 2");
    if (cfg->beams < 1 || (3 * cfg->beams) % 4 != 0)
        return rlca_set_err(RLCA_ERR_UNSUPPORTED, "rlca_demo_append: 3 * beams must be a multiple of 4");
    if (!io->stack_in_dev || !io->gs_dev || !io->action_dev || !demo->obs_dev || !demo->gs_dev || !demo->action_dev ||
        !demo->count_dev || (cfg->auto_reset == 2 && !state->meta_dev))
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_demo_append: a buffer is NULL");
    if (io->live_dev) return rlca_set_err(RLCA_ERR_UNSUPPORTED, "rlca_demo_append: a live mask is not supported");
    if (demo->capacity < 1) return rlca_set_err(RLCA_ERR_INVALID, "rlca_demo_append: capacity must be >= 1");
    if ((((uintptr_t)io->stack_in_dev | (uintptr_t)io->gs_dev | (uintptr_t)demo->obs_dev | (uintptr_t)demo->gs_dev) & 15) ||
        (((uintptr_t)io->action_dev | (uintptr_t)demo->action_dev) & 7) || ((uintptr_t)demo->count_dev & 7))
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_demo_append: misaligned buffer");
    if (!(cfg->v_min <= cfg->v_max) || !(cfg->w_min <= cfg->w_max))
        return rlca_set_err(RLCA_ERR_INVALID, "cfg action bounds are empty");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const int ctas = (n + DEMO_AGENTS - 1) / DEMO_AGENTS;
    demo_append_kernel<<<ctas, DEMO_THREADS, 0, (cudaStream_t)stream>>>(
        n, cfg->auto_reset, 3 * cfg->beams / 4, cfg->v_min, cfg->v_max, cfg->w_min, cfg->w_max,
        reinterpret_cast<const float4 *>(io->stack_in_dev), reinterpret_cast<const float4 *>(io->gs_dev),
        reinterpret_cast<const float2 *>(io->action_dev), reinterpret_cast<const int4 *>(state->meta_dev),
        io->flags_dev, reinterpret_cast<float4 *>(demo->obs_dev), reinterpret_cast<float4 *>(demo->gs_dev),
        reinterpret_cast<float2 *>(demo->action_dev), reinterpret_cast<unsigned long long *>(demo->count_dev),
        (long long)demo->capacity);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}
