// rlca_dp.cu — data-parallel optimizer step fused with its collective, over NVLink peer memory (sm_90a).
//
// The reference takes an Adam step per minibatch (model/ppo.py:186-188), so under data parallelism the gradient
// all-reduce sits on the critical path of every step.  Instead of NCCL all-reduce (8.69 MB) followed by the Adam
// kernel, ONE kernel does reduce-scatter + Adam + all-gather through peer mappings of the other GPUs' buffers:
//
//   rank r owns the elements [r * chunk, (r + 1) * chunk) of the flat buffer.  For each of them it
//     sums the gradient over all ranks   - plain loads from the W peer mappings, or one multimem.ld_reduce.add on the
//                                          NVSwitch multicast mapping (the switch does the sum in flight, NVLS);
//     applies Adam                       - same arithmetic and rounding as adam_kernel (torch.optim.Adam semantics);
//     writes the new parameter into EVERY rank's buffer - W peer stores, or one multimem.st (the switch replicates it);
//     keeps the two moments of its shard locally (the optimizer state is sharded: a checkpoint reads the shards back
//     through the peer mappings), or - replicate_moments - writes them everywhere too (3x the outbound traffic).
//
// Every rank therefore ends with bit-identical parameters, having moved 1/W of the gradient in and 1/W of the
// parameters out per peer.  The caller brackets the launch with
// two cross-GPU barriers (all gradients complete before / all shards written after); buffers and barriers come from a
// symmetric-memory allocation (PyTorch's, which is plumbing here: cuMemCreate + peer mapping + multicast binding).
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define DP_MAX_RANKS 16

struct DpPtrs {
    float *grad[DP_MAX_RANKS];
    float *param[DP_MAX_RANKS];
    float *m[DP_MAX_RANKS];
    float *v[DP_MAX_RANKS];
    float *mc_grad, *mc_param, *mc_m, *mc_v;      // multicast mappings of the same buffers, or NULL
};

__device__ __forceinline__ float4 mm_ld_reduce_add(const float *p)
{
    float4 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
}

__device__ __forceinline__ void mm_st(float *p, float4 v)
{
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}

template <bool NVLS, bool REPL>
__global__ void __launch_bounds__(256) adam_allreduce_kernel(const __grid_constant__ DpPtrs P, int rank, int world,
                                                             int64_t lo, int64_t hi, float lr, float b1, float b2,
                                                             float eps, float bc1, float bc2_sqrt, float grad_scale)
{
    // elements [lo, hi) of the flat buffer, lo and hi multiples of 4 (the buffer is padded to 32 floats per tensor)
    const int64_t n4 = (hi - lo) >> 2;
    for (int64_t i4 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = lo + (i4 << 2);
        float4 g;
        if (NVLS) {
            g = mm_ld_reduce_add(P.mc_grad + i);
        } else {
            g = *reinterpret_cast<const float4 *>(P.grad[0] + i);
            for (int q = 1; q < world; ++q) {                  // fixed order: every rank would get the same sum
                const float4 t = *reinterpret_cast<const float4 *>(P.grad[q] + i);
                g.x += t.x; g.y += t.y; g.z += t.z; g.w += t.w;
            }
        }
        const float4 pm = *reinterpret_cast<const float4 *>(P.m[rank] + i);
        const float4 pv = *reinterpret_cast<const float4 *>(P.v[rank] + i);
        const float4 pp = *reinterpret_cast<const float4 *>(P.param[rank] + i);
        float gi[4] = { g.x, g.y, g.z, g.w }, mi[4] = { pm.x, pm.y, pm.z, pm.w }, vi[4] = { pv.x, pv.y, pv.z, pv.w },
              pi[4] = { pp.x, pp.y, pp.z, pp.w };
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float gk = gi[k] * grad_scale;
            mi[k] = fmaf(b1, mi[k], (1.0f - b1) * gk);
            vi[k] = fmaf(b2, vi[k], (1.0f - b2) * gk * gk);
            // torch.optim.Adam: denom = sqrt(v)/sqrt(bias_correction2) + eps ; p -= lr/bias_correction1 * m/denom
            const float denom = sqrtf(vi[k]) / bc2_sqrt + eps;
            pi[k] -= (lr / bc1) * (mi[k] / denom);
        }
        const float4 nm = make_float4(mi[0], mi[1], mi[2], mi[3]), nv = make_float4(vi[0], vi[1], vi[2], vi[3]),
                     np = make_float4(pi[0], pi[1], pi[2], pi[3]);
        if (NVLS) {
            mm_st(P.mc_param + i, np);
            if (REPL) { mm_st(P.mc_m + i, nm); mm_st(P.mc_v + i, nv); }
        } else {
            for (int q = 0; q < world; ++q) {
                *reinterpret_cast<float4 *>(P.param[q] + i) = np;
                if (REPL) {
                    *reinterpret_cast<float4 *>(P.m[q] + i) = nm;
                    *reinterpret_cast<float4 *>(P.v[q] + i) = nv;
                }
            }
        }
        if (!REPL) {
            *reinterpret_cast<float4 *>(P.m[rank] + i) = nm;
            *reinterpret_cast<float4 *>(P.v[rank] + i) = nv;
        }
    }
}

extern "C" int rlca_adam_step_allreduce(const uint64_t *grad_ptrs, const uint64_t *param_ptrs, const uint64_t *m_ptrs,
                                        const uint64_t *v_ptrs, uint64_t mc_grad, uint64_t mc_param, uint64_t mc_m,
                                        uint64_t mc_v, int32_t rank, int32_t world, int64_t n, float lr, float beta1,
                                        float beta2, float eps, int32_t step, float grad_scale, int32_t replicate_moments,
                                        void *stream)
{
    if (!grad_ptrs || !param_ptrs || !m_ptrs || !v_ptrs || world < 1 || world > DP_MAX_RANKS || rank < 0 || rank >= world ||
        n < 1 || (n & 3) || step < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "bad rlca_adam_step_allreduce arguments (1 <= world <= 16, n % 4 == 0)");
    DpPtrs P{};
    for (int q = 0; q < world; ++q) {
        P.grad[q] = reinterpret_cast<float *>(grad_ptrs[q]);
        P.param[q] = reinterpret_cast<float *>(param_ptrs[q]);
        P.m[q] = reinterpret_cast<float *>(m_ptrs[q]);
        P.v[q] = reinterpret_cast<float *>(v_ptrs[q]);
        if (!P.grad[q] || !P.param[q] || !P.m[q] || !P.v[q]) return rlca_set_err(RLCA_ERR_INVALID, "NULL peer pointer");
    }
    P.mc_grad = reinterpret_cast<float *>(mc_grad);
    P.mc_param = reinterpret_cast<float *>(mc_param);
    P.mc_m = reinterpret_cast<float *>(mc_m);
    P.mc_v = reinterpret_cast<float *>(mc_v);
    const bool nvls = mc_grad && mc_param && mc_m && mc_v;
    // shard: n / world elements rounded up to 4 floats
    const int64_t chunk = ((n / 4 + world - 1) / world) * 4;
    const int64_t lo = (int64_t)rank * chunk < n ? (int64_t)rank * chunk : n;
    const int64_t hi = lo + chunk < n ? lo + chunk : n;
    const float bc1 = 1.0f - powf(beta1, (float)step);
    const float bc2 = 1.0f - powf(beta2, (float)step);
    if (hi > lo) {
        const int64_t n4 = (hi - lo) >> 2;
        unsigned blocks = (unsigned)((n4 + 255) / 256);
        if (blocks > 592u) blocks = 592u;                       // 4 CTAs per SM: the kernel is bound by the links
#define DP_LAUNCH(NV, RP) adam_allreduce_kernel<NV, RP><<<blocks, 256, 0, (cudaStream_t)stream>>>( \
            P, rank, world, lo, hi, lr, beta1, beta2, eps, bc1, sqrtf(bc2), grad_scale)
        if (nvls && replicate_moments) DP_LAUNCH(true, true);
        else if (nvls) DP_LAUNCH(true, false);
        else if (replicate_moments) DP_LAUNCH(false, true);
        else DP_LAUNCH(false, false);
#undef DP_LAUNCH
        RLCA_CUDA_TRY(cudaGetLastError());
    }
    return RLCA_OK;
}
