// rlca_policy.cu — CNNPolicy forward/backward, PPO loss, GAE, Adam for sm_90a (C ABI in include/rlca.h).
//
// Round-1 layout of the learner: every op is a hand-written CUDA kernel (no cuDNN/cuBLAS/ATen):
//   conv tower   fused conv1+ReLU+conv2+ReLU per (sample, tower), activations in shared memory
//   fc1 / fc2    tiled fp32 GEMM with fused bias / ReLU / mask epilogues (fc1 has a wgmma path in
//                rlca_gemm_tc.cu when enabled)
//   heads, sampling, PPO loss (+ its gradient), GAE (float64 recurrence), Adam: fused elementwise/reduction kernels
// Parameters, gradients and Adam moments are flat fp32 buffers in state_dict order (tensor starts
// padded to 32 floats so every matrix is 128-byte aligned).
#include <cuda_runtime.h>
#include <stdlib.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>
#include <new>

#include "../../include/rlca.h"
#include "rlca_common.cuh"
#include "rlca_gemm_tc.cuh"
#include "rlca_conv_tc.cuh"

// ------------------------------------------------------------------------------------ layout
static const int64_t kTensorSize[RLCA_POLICY_NTENSORS] = {
    2, 480, 32, 3072, 32, 1048576, 256, 33280, 128, 128, 1, 128, 1,
    480, 32, 3072, 32, 1048576, 256, 33280, 128, 128, 1};

static int64_t tensor_offset(int i)
{
    int64_t off = 0;
    for (int k = 0; k < i && k < RLCA_POLICY_NTENSORS; ++k) off += (kTensorSize[k] + 31) / 32 * 32;
    return off;
}

extern "C" int64_t rlca_policy_param_offset(int32_t i)
{
    if (i < 0) return -1;
    if (i >= RLCA_POLICY_NTENSORS) return tensor_offset(RLCA_POLICY_NTENSORS);
    return tensor_offset(i);
}
extern "C" int64_t rlca_policy_param_size(int32_t i)
{
    return (i >= 0 && i < RLCA_POLICY_NTENSORS) ? kTensorSize[i] : -1;
}

enum { T_LOGSTD = 0, T_CV1W = 1, T_CV1B, T_CV2W, T_CV2B, T_FC1W, T_FC1B, T_FC2W, T_FC2B, T_A1W, T_A1B, T_A2W, T_A2B,
       T_CRT0 = 13, T_CRITW = 21, T_CRITB = 22 };

struct TowerPtrs {
    const float *cv1w, *cv1b, *cv2w, *cv2b, *fc1w, *fc1b, *fc2w, *fc2b;
};
struct TowerGrads {
    float *cv1w, *cv1b, *cv2w, *cv2b, *fc1w, *fc1b, *fc2w, *fc2b;
};

static TowerPtrs tower_ptrs(const float *p, int tower)
{
    const int b = tower == 0 ? T_CV1W : T_CRT0;
    TowerPtrs t;
    t.cv1w = p + tensor_offset(b + 0); t.cv1b = p + tensor_offset(b + 1);
    t.cv2w = p + tensor_offset(b + 2); t.cv2b = p + tensor_offset(b + 3);
    t.fc1w = p + tensor_offset(b + 4); t.fc1b = p + tensor_offset(b + 5);
    t.fc2w = p + tensor_offset(b + 6); t.fc2b = p + tensor_offset(b + 7);
    return t;
}
static TowerGrads tower_grads(float *p, int tower)
{
    const int b = tower == 0 ? T_CV1W : T_CRT0;
    TowerGrads t;
    t.cv1w = p + tensor_offset(b + 0); t.cv1b = p + tensor_offset(b + 1);
    t.cv2w = p + tensor_offset(b + 2); t.cv2b = p + tensor_offset(b + 3);
    t.fc1w = p + tensor_offset(b + 4); t.fc1b = p + tensor_offset(b + 5);
    t.fc2w = p + tensor_offset(b + 6); t.fc2b = p + tensor_offset(b + 7);
    return t;
}

#define FEAT 4096
#define XLD 260          // fc2 input: 256 fc1 outputs + goal(2) + speed(2)
#define RSPLIT 16        // row/K splits of the small batch reductions (two-stage, deterministic)
#define CONV_PART 3616   // per-(sample,tower) conv gradient partials: cv2w 3072 | cv2b 32 | cv1w 480 | cv1b 32

struct rlca_policy {
    int max_batch;
    float *F;        // [2][B][4096] relu(conv2) features, flatten order c*128+p (model/net.py:44)
    float *X;        // [2][B][260]  relu(fc1) | goal | speed
    float *H2;       // [2][B][128]  relu(fc2)
    float *dOut;     // [B][4]  dL/dv, dL/dz1, dL/dz2, unused
    float *dZ2;      // [2][B][128]
    float *dX;       // [2][B][260]  (masked in place -> dZ1 in the first 256 columns)
    float *dF;       // [2][B][4096]
    float *part;     // [2][B][CONV_PART]
    float *headpart; // [chunks][3][128 + 4]
    float *red;      // small reduction scratch (64 floats)
    float *Wc;       // prepared conv weights [2][CONV_WBLK] (transposed for conflict-free staging)
    float *S;        // split-reduction scratch: [RSPLIT][2][max(CONV_PART, 128*260)]
    // ---- tensor-core (3xTF32) path for fc1: hi/lo splits of the operands, all K-major
    int use_tc;
    int weights_dirty;   // W1 hi/lo/transposed copies must be rebuilt at the next forward
    int wimg_dirty;      // Wimg must be rebuilt before the tensor-core conv tower forward runs next
    int bpad;        // max_batch rounded up to 32 (row pitch of the transposed operands)
    float *Fs;       // [2 towers][hi,lo][B][4096]
    float *W1s;      // [2][hi,lo][256][4096]
    float *W1Ts;     // [2][hi,lo][4096][256]
    float *dZs;      // [2][hi,lo][B][256]
    float *dZTs;     // [2][hi,lo][256][bpad]
    float *FTs;      // [2][hi,lo][4096][bpad]
    float *P;        // split-K partials [splits<=8][2][B][256]
    int use_tc_conv; // conv tower on wgmma (rlca_conv_tc.cu); needs use_tc (it feeds the fc1 GEMM's hi/lo split)
    int num_sms;
    float *Wimg;     // pre-swizzled tf32 hi/lo image of the conv weights for the tensor-core conv tower
    float *WimgB;    // same for the backward kernel (per tower: conv1 weights | conv2 weights regrouped by tap)
    int conv_bwd_dirty;
    int wc_dirty;        // Wc (the CUDA-core conv kernels' weight block) is rebuilt only when one of them is about to run
    int w1_split_valid;  // W1s / W1Ts already hold the current fc1 weights (written by rlca_policy_adam_step)
    cudaEvent_t fc_grads_event;   // optional: recorded by rlca_policy_backward once every gradient outside the conv towers is final
    int reserved_sms;             // SMs the persistent conv tower backward leaves free while that event is set (for the collective)
    // ---- side streams of the backward: the work that is not on the chain heads -> dX -> dF -> conv towers (transposed
    // split of F, every weight / bias gradient of the fc layers and the heads) runs beside it
    int use_side;                 // 0: one stream (RLCA_BWD_STREAMS=0, or while fc_grads_event is set)
    cudaStream_t side[2];
    cudaEvent_t ev_fork, ev_heads, ev_dx, ev_split, ev_prep, ev_join[2];
    float *S2;                    // split-reduction scratch of the conv tower partials (the side streams use S meanwhile)
    int64_t launches;
};

// ------------------------------------------------------------------------------------ conv tower forward
// One CTA per sample; threads 0..127 run the actor tower, 128..255 the critic tower.
// conv1: Conv1d(3,32,k5,s2,p1) 512 -> 255 ; conv2: Conv1d(32,32,k3,s2,p1) 255 -> 128 (model/net.py:21-22,42-43).
// h1 is kept in shared memory split into even/odd positions so conv2's stride-2 reads are conflict free:
// stored index s = q+1 (q = -1..255, zeros at both ends); even s -> h1e[s/2], odd s -> h1o[s/2].  The input scan is
// split the same way (xe/xo) for conv1's stride-2 reads, and h1o is skewed by 16 floats so that the conv1 stores of
// one warp (alternating even/odd s) spread over all 32 banks.
// Weights come from a pre-transposed block Wc[tower] = w1t[15][32] | b1[32] | w2t[96][32] | b2[32] built by
// conv_prep_weights_kernel, so staging them is a conflict-free linear copy (an in-kernel transpose would cause
// shared-memory bank conflicts).
#define CONV_WBLK 3616          // floats per tower in the prepared weight block
#define CONV_SPC 4              // samples per CTA: amortises the 29 KB weight staging
struct ConvSmem {
    float wc[2][CONV_WBLK];      // [tower]: w1t | b1 | w2t | b2
    float xe[3][264], xo[3][264];   // x de-interleaved: padded index j = i+1 (j = 0..513); even j -> xe[j/2], odd -> xo[j/2]
    float h1e[2][32][132];
    float skew[16];
    float h1o[2][32][132];
};
#define WC_W1(sm, t, j) (&(sm).wc[t][(j) * 32])
#define WC_B1(sm, t) (&(sm).wc[t][480])
#define WC_W2(sm, t, j) (&(sm).wc[t][512 + (j) * 32])
#define WC_B2(sm, t) (&(sm).wc[t][512 + 3072])

// Wc[t] from the state_dict layouts (co, ci, k): w1t[ci*5+k][co], w2t[ci*3+k][co]
__global__ void conv_prep_weights_kernel(TowerPtrs ta, TowerPtrs tc, float *__restrict__ Wc)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
    if (i >= CONV_WBLK) return;
    const TowerPtrs &tp = t == 0 ? ta : tc;
    float v;
    if (i < 480) { const int j = i >> 5, co = i & 31; v = tp.cv1w[co * 15 + j]; }
    else if (i < 512) v = tp.cv1b[i - 480];
    else if (i < 512 + 3072) { const int r = i - 512, j = r >> 5, co = r & 31; v = tp.cv2w[co * 96 + j]; }
    else v = tp.cv2b[i - 3584];
    Wc[(size_t)t * CONV_WBLK + i] = v;
}

__device__ __forceinline__ void conv_stage_weights(ConvSmem &sm, const float *__restrict__ Wc, int tid, int nthreads)
{
    const float4 *src = reinterpret_cast<const float4 *>(Wc);
    float4 *dst = reinterpret_cast<float4 *>(&sm.wc[0][0]);
    for (int i = tid; i < 2 * CONV_WBLK / 4; i += nthreads) dst[i] = src[i];
    for (int i = tid; i < 2 * 32; i += nthreads) {
        int t = i >> 5, c = i & 31;
        sm.h1e[t][c][0] = 0.0f;        // s = 0   (q = -1)
        sm.h1e[t][c][128] = 0.0f;      // s = 256 (q = 255)
    }
}

__device__ __forceinline__ void conv_stage_x(ConvSmem &sm, const float *__restrict__ obs_n, int tid, int nthreads)
{
    // padded index j = i + 1; j = 0 and j >= 513 are the zero padding of Conv1d(padding=1)
    for (int i = tid; i < 3 * 264; i += nthreads) {
        const int c = i / 264, h = i - c * 264;
        const int je = 2 * h, jo = 2 * h + 1;
        sm.xe[c][h] = (je >= 1 && je <= 512) ? obs_n[c * 512 + je - 1] : 0.0f;
        sm.xo[c][h] = (jo >= 1 && jo <= 512) ? obs_n[c * 512 + jo - 1] : 0.0f;
    }
}

// conv1 + ReLU for one tower by 128 threads (lt = 0..127): positions lt and lt+128.
__device__ __forceinline__ void conv1_tower(ConvSmem &sm, int t, int lt)
{
#pragma unroll 1
    for (int rep = 0; rep < 2; ++rep) {
        const int p = lt + rep * 128;
        if (p >= 255) break;
        float xv[15];
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {          // padded input index 2p+k: k even -> xe[p + k/2], k odd -> xo[p + k/2]
            xv[ci * 5 + 0] = sm.xe[ci][p];
            xv[ci * 5 + 1] = sm.xo[ci][p];
            xv[ci * 5 + 2] = sm.xe[ci][p + 1];
            xv[ci * 5 + 3] = sm.xo[ci][p + 1];
            xv[ci * 5 + 4] = sm.xe[ci][p + 2];
        }
        const int s = p + 1;
        float *dst = (s & 1) ? &sm.h1o[t][0][s >> 1] : &sm.h1e[t][0][s >> 1];
#pragma unroll
        for (int cg = 0; cg < 8; ++cg) {
            float4 acc = *reinterpret_cast<const float4 *>(WC_B1(sm, t) + cg * 4);
#pragma unroll
            for (int j = 0; j < 15; ++j) {
                const float4 w = *reinterpret_cast<const float4 *>(WC_W1(sm, t, j) + cg * 4);
                acc.x = fmaf(xv[j], w.x, acc.x); acc.y = fmaf(xv[j], w.y, acc.y);
                acc.z = fmaf(xv[j], w.z, acc.z); acc.w = fmaf(xv[j], w.w, acc.w);
            }
            dst[(cg * 4 + 0) * 132] = fmaxf(acc.x, 0.0f);
            dst[(cg * 4 + 1) * 132] = fmaxf(acc.y, 0.0f);
            dst[(cg * 4 + 2) * 132] = fmaxf(acc.z, 0.0f);
            dst[(cg * 4 + 3) * 132] = fmaxf(acc.w, 0.0f);
        }
    }
}

__global__ void __launch_bounds__(256) conv_tower_fwd_kernel(const float *__restrict__ obs, const float *__restrict__ Wc,
                                                             float *__restrict__ F, float *__restrict__ Fs, int nb)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    ConvSmem &sm = *reinterpret_cast<ConvSmem *>(smem_raw);
    const int tid = threadIdx.x;
    const int t = tid >> 7, lt = tid & 127;
    const int pg = lt & 31, cg = lt >> 5;
    conv_stage_weights(sm, Wc, tid, 256);
    for (int rep = 0; rep < CONV_SPC; ++rep) {
        const int n = blockIdx.x * CONV_SPC + rep;
        if (n >= nb) break;
        if (rep) __syncthreads();                 // previous sample's conv2 has finished reading h1 / x
        conv_stage_x(sm, obs + (size_t)n * 1536, tid, 256);
        __syncthreads();
        conv1_tower(sm, t, lt);
        __syncthreads();
        // conv2: thread = 4 consecutive positions (4 pg .. 4 pg + 3) x 8 channels (cg*8 ..): the three taps of the four
        // positions need h1e[4pg .. 4pg+4] and h1o[4pg .. 4pg+3] -> two LDS.128 + one LDS.32 per input channel
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[i][c] = WC_B2(sm, t)[cg * 8 + c];
#pragma unroll 2
        for (int ci = 0; ci < 32; ++ci) {
            const float4 e = *reinterpret_cast<const float4 *>(&sm.h1e[t][ci][4 * pg]);
            const float e4 = sm.h1e[t][ci][4 * pg + 4];
            const float4 o = *reinterpret_cast<const float4 *>(&sm.h1o[t][ci][4 * pg]);
            const float a0[4] = {e.x, e.y, e.z, e.w};          // k = 0: s = 2p
            const float a1[4] = {o.x, o.y, o.z, o.w};          // k = 1: s = 2p+1
            const float a2[4] = {e.y, e.z, e.w, e4};           // k = 2: s = 2p+2
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float4 wa = *reinterpret_cast<const float4 *>(WC_W2(sm, t, ci * 3 + k) + cg * 8);
                const float4 wb = *reinterpret_cast<const float4 *>(WC_W2(sm, t, ci * 3 + k) + cg * 8 + 4);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float a = k == 0 ? a0[i] : (k == 1 ? a1[i] : a2[i]);
                    acc[i][0] = fmaf(a, wa.x, acc[i][0]); acc[i][1] = fmaf(a, wa.y, acc[i][1]);
                    acc[i][2] = fmaf(a, wa.z, acc[i][2]); acc[i][3] = fmaf(a, wa.w, acc[i][3]);
                    acc[i][4] = fmaf(a, wb.x, acc[i][4]); acc[i][5] = fmaf(a, wb.y, acc[i][5]);
                    acc[i][6] = fmaf(a, wb.z, acc[i][6]); acc[i][7] = fmaf(a, wb.w, acc[i][7]);
                }
            }
        }
        float *out = F + ((size_t)t * nb + n) * FEAT;
        // optional tf32 hi/lo split of the features for the tensor-core fc1 (Fs = [tower][hi,lo][nb][4096])
        float *out_hi = Fs ? Fs + ((size_t)(2 * t) * nb + n) * FEAT : nullptr;
        float *out_lo = Fs ? Fs + ((size_t)(2 * t + 1) * nb + n) * FEAT : nullptr;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int o = (cg * 8 + c) * 128 + 4 * pg;
            const float4 v = make_float4(fmaxf(acc[0][c], 0.0f), fmaxf(acc[1][c], 0.0f), fmaxf(acc[2][c], 0.0f),
                                         fmaxf(acc[3][c], 0.0f));
            *reinterpret_cast<float4 *>(out + o) = v;
            if (Fs) {
                float4 h;
                h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u); h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
                h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u); h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
                *reinterpret_cast<float4 *>(out_hi + o) = h;
                *reinterpret_cast<float4 *>(out_lo + o) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
            }
        }
    }
}

// ------------------------------------------------------------------------------------ conv tower backward
// One CTA per (CONV_SPC samples, tower), 256 threads.  dF is d(relu(conv2)) - masked here by Fmask > 0, or already
// masked by the producing GEMM when Fmask is NULL.
// Shared-memory layouts are chosen so that every hot loop reads conflict-free or by broadcast:
//   g2t[p][co] / g1t[s][co]  position-major with pitch 33 (lanes over co: consecutive; lanes over p: stride 33)
//   h1e / h1o                channel-major even/odd split as in the forward kernel (read by broadcast here)
//   w2c[co][ci*3+k]          the state_dict layout (12 consecutive weights per (co, 4 ci) -> 3 broadcast LDS.128)
struct ConvBwdSmem {
    float w1[15][32];            // w1t from the prepared block
    float b1[32];
    float w2c[32][96];
    float xe[3][264], xo[3][264];
    float h1e[32][132];
    float skew[16];
    float h1o[32][132];
    float g2t[129][33];          // d conv2 pre-activation, row 128 = 0; reused as the dW1 reduction scratch
    float g1t[257][33];          // d conv1 pre-activation at stored index s = q+1 (rows 0 and 256 unused)
};

__global__ void __launch_bounds__(256) conv_tower_bwd_kernel(const float *__restrict__ obs, const float *__restrict__ Wc,
                                                             TowerPtrs ta, TowerPtrs tc, const float *__restrict__ dF,
                                                             const float *__restrict__ Fmask,
                                                             float *__restrict__ part, int nb)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    ConvBwdSmem &sm = *reinterpret_cast<ConvBwdSmem *>(smem_raw);
    const int t = blockIdx.y, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const TowerPtrs &tp = t == 0 ? ta : tc;
    {   // weights: w1t | b1 from the prepared block, conv2 weights in their native (co, ci, k) order
        const float4 *src = reinterpret_cast<const float4 *>(Wc + (size_t)t * CONV_WBLK);
        float4 *dst = reinterpret_cast<float4 *>(&sm.w1[0][0]);
        for (int i = tid; i < 512 / 4; i += 256) dst[i] = src[i];
        const float4 *src2 = reinterpret_cast<const float4 *>(tp.cv2w);
        float4 *dst2 = reinterpret_cast<float4 *>(&sm.w2c[0][0]);
        for (int i = tid; i < 3072 / 4; i += 256) dst2[i] = src2[i];
        if (tid < 32) { sm.h1e[tid][0] = 0.f; sm.h1e[tid][128] = 0.f; }
    }
    for (int rep = 0; rep < CONV_SPC; ++rep) {
        const int n = blockIdx.x * CONV_SPC + rep;
        if (n >= nb) break;
        __syncthreads();
        const float *obs_n = obs + (size_t)n * 1536;
        for (int i = tid; i < 3 * 264; i += 256) {
            const int c = i / 264, h = i - c * 264;
            const int je = 2 * h, jo = 2 * h + 1;
            sm.xe[c][h] = (je >= 1 && je <= 512) ? obs_n[c * 512 + je - 1] : 0.0f;
            sm.xo[c][h] = (jo >= 1 && jo <= 512) ? obs_n[c * 512 + jo - 1] : 0.0f;
        }
        const float *dF_n = dF + ((size_t)t * nb + n) * FEAT;
        // coalesced read, stride-33 write; the relu(conv2) mask is applied here when the dF GEMM left it to us
        if (Fmask) {
            const float *F_n = Fmask + ((size_t)t * nb + n) * FEAT;
            for (int i = tid; i < 4096; i += 256) sm.g2t[i & 127][i >> 7] = F_n[i] > 0.0f ? dF_n[i] : 0.0f;
        } else {
            for (int i = tid; i < 4096; i += 256) sm.g2t[i & 127][i >> 7] = dF_n[i];
        }
        if (tid < 33) sm.g2t[128][tid] = 0.0f;
        __syncthreads();
        // ---- recompute h1 = relu(conv1(x)): thread = position (255 of them)
        if (tid < 255) {
            const int p = tid;
            float xv[15];
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) {
                xv[ci * 5 + 0] = sm.xe[ci][p];     xv[ci * 5 + 1] = sm.xo[ci][p];
                xv[ci * 5 + 2] = sm.xe[ci][p + 1]; xv[ci * 5 + 3] = sm.xo[ci][p + 1];
                xv[ci * 5 + 4] = sm.xe[ci][p + 2];
            }
            const int s = p + 1;
            float *dst = (s & 1) ? &sm.h1o[0][s >> 1] : &sm.h1e[0][s >> 1];
#pragma unroll
            for (int cg = 0; cg < 8; ++cg) {
                float4 acc = *reinterpret_cast<const float4 *>(&sm.b1[cg * 4]);
#pragma unroll
                for (int j = 0; j < 15; ++j) {
                    const float4 w = *reinterpret_cast<const float4 *>(&sm.w1[j][cg * 4]);
                    acc.x = fmaf(xv[j], w.x, acc.x); acc.y = fmaf(xv[j], w.y, acc.y);
                    acc.z = fmaf(xv[j], w.z, acc.z); acc.w = fmaf(xv[j], w.w, acc.w);
                }
                dst[(cg * 4 + 0) * 132] = fmaxf(acc.x, 0.0f);
                dst[(cg * 4 + 1) * 132] = fmaxf(acc.y, 0.0f);
                dst[(cg * 4 + 2) * 132] = fmaxf(acc.z, 0.0f);
                dst[(cg * 4 + 3) * 132] = fmaxf(acc.w, 0.0f);
            }
        }
        __syncthreads();
        float *out = part + ((size_t)t * nb + n) * CONV_PART;
        // ---- (a) dW2[co][ci][k] = sum_p g2[co][p] h1[ci][2p+k-1]: lane = co, warp = 4 input channels
        {
            const int co = lane, ci0 = warp * 4;
            float acc[4][3];
#pragma unroll
            for (int a = 0; a < 4; ++a) acc[a][0] = acc[a][1] = acc[a][2] = 0.0f;
            float bsum = 0.0f;
            for (int p = 0; p < 128; p += 4) {
                const float g0 = sm.g2t[p][co], g1v = sm.g2t[p + 1][co], g2v = sm.g2t[p + 2][co], g3 = sm.g2t[p + 3][co];
                bsum += (g0 + g1v) + (g2v + g3);
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    const float4 e = *reinterpret_cast<const float4 *>(&sm.h1e[ci0 + a][p]);     // broadcast
                    const float e4 = sm.h1e[ci0 + a][p + 4];
                    const float4 o = *reinterpret_cast<const float4 *>(&sm.h1o[ci0 + a][p]);
                    acc[a][0] = fmaf(g0, e.x, fmaf(g1v, e.y, fmaf(g2v, e.z, fmaf(g3, e.w, acc[a][0]))));
                    acc[a][1] = fmaf(g0, o.x, fmaf(g1v, o.y, fmaf(g2v, o.z, fmaf(g3, o.w, acc[a][1]))));
                    acc[a][2] = fmaf(g0, e.y, fmaf(g1v, e.z, fmaf(g2v, e.w, fmaf(g3, e4, acc[a][2]))));
                }
            }
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int k = 0; k < 3; ++k) out[co * 96 + (ci0 + a) * 3 + k] = acc[a][k];
            if (warp == 0) out[3072 + co] = bsum;                     // (b) db2[co] = sum_p g2[co][p]
        }
        // ---- (c) dh1[ci][q] = sum_co sum_k g2[co][p] w2[co][ci][k], q = 2p+k-1, masked by h1 > 0
        //      item = (m = 0..127, 4 input channels): q = 2m (k=1, p=m) and q = 2m+1 (k=0, p=m+1 ; k=2, p=m)
        {   // thread = (positions lane + 32 j, j = 0..3 ; 4 input channels): 8 conflict-free g loads (pitch 33) + 3 broadcast
            // weight LDS.128 per co for 48 FMAs
            const int ml = tid & 31, ci0 = (tid >> 5) * 4;
            float ev[4][4], od[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int a = 0; a < 4; ++a) ev[j][a] = od[j][a] = 0.0f;
#pragma unroll 2
            for (int co = 0; co < 32; ++co) {
                float g[4], gn[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) { g[j] = sm.g2t[ml + 32 * j][co]; gn[j] = sm.g2t[ml + 32 * j + 1][co]; }   // row 128 is zero
                const float4 wa = *reinterpret_cast<const float4 *>(&sm.w2c[co][ci0 * 3]);       // broadcast
                const float4 wb = *reinterpret_cast<const float4 *>(&sm.w2c[co][ci0 * 3 + 4]);
                const float4 wc = *reinterpret_cast<const float4 *>(&sm.w2c[co][ci0 * 3 + 8]);
                const float w[12] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w, wc.x, wc.y, wc.z, wc.w};
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int a = 0; a < 4; ++a) {
                        ev[j][a] = fmaf(g[j], w[a * 3 + 1], ev[j][a]);
                        od[j][a] = fmaf(gn[j], w[a * 3 + 0], fmaf(g[j], w[a * 3 + 2], od[j][a]));
                    }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int m = ml + 32 * j;
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    // q = 2m -> s = 2m+1 ; q = 2m+1 -> s = 2m+2 (q = 255 does not exist)
                    sm.g1t[2 * m + 1][ci0 + a] = sm.h1o[ci0 + a][m] > 0.0f ? ev[j][a] : 0.0f;
                    if (m < 127) sm.g1t[2 * m + 2][ci0 + a] = sm.h1e[ci0 + a][m + 1] > 0.0f ? od[j][a] : 0.0f;
                }
            }
        }
        __syncthreads();
        // ---- (d) dW1[co][ci][k] = sum_p g1[co][p] x[ci][2p+k-1], db1[co] = sum_p g1[co][p]  (p = 0..254, s = p+1):
        //      lane = co, warp w takes positions p = w, w+8, ...; 16 partial sums per thread, reduced across warps
        {
            const int co = lane;
            float acc[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j] = 0.0f;
            for (int p = warp; p < 255; p += 8) {
                const float g = sm.g1t[p + 1][co];
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    acc[ci * 5 + 0] = fmaf(g, sm.xe[ci][p], acc[ci * 5 + 0]);
                    acc[ci * 5 + 1] = fmaf(g, sm.xo[ci][p], acc[ci * 5 + 1]);
                    acc[ci * 5 + 2] = fmaf(g, sm.xe[ci][p + 1], acc[ci * 5 + 2]);
                    acc[ci * 5 + 3] = fmaf(g, sm.xo[ci][p + 1], acc[ci * 5 + 3]);
                    acc[ci * 5 + 4] = fmaf(g, sm.xe[ci][p + 2], acc[ci * 5 + 4]);
                }
                acc[15] += g;
            }
            float *red = &sm.g2t[0][0];                 // g2t is dead after (c): [warp][16][32] = 4096 floats <= 129*33
#pragma unroll
            for (int j = 0; j < 16; ++j) red[(warp * 16 + j) * 32 + co] = acc[j];
        }
        __syncthreads();
        for (int o = tid; o < 512; o += 256) {
            const int j = o >> 5, co = o & 31;
            const float *red = &sm.g2t[0][0];
            float v = 0.0f;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += red[(w * 16 + j) * 32 + co];
            if (j < 15) out[3104 + co * 15 + j] = v;
            else out[3104 + 480 + co] = v;
        }
    }
}

// sum the per-sample conv partials over the batch: grid (ceil(CONV_PART/256), 2)
__global__ void conv_part_reduce_kernel(const float *__restrict__ part, int nb, float *__restrict__ P)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
    if (j >= CONV_PART) return;
    const int nper = (nb + gridDim.z - 1) / gridDim.z;
    const int nbeg = blockIdx.z * nper, nend = min(nb, nbeg + nper);
    const float *src = part + (size_t)t * nb * CONV_PART + j;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int n = nbeg;
    nb = nend;
    for (; n + 3 < nb; n += 4) {
        a0 += src[(size_t)(n + 0) * CONV_PART]; a1 += src[(size_t)(n + 1) * CONV_PART];
        a2 += src[(size_t)(n + 2) * CONV_PART]; a3 += src[(size_t)(n + 3) * CONV_PART];
    }
    for (; n < nb; ++n) a0 += src[(size_t)n * CONV_PART];
    P[((size_t)blockIdx.z * 2 + t) * CONV_PART + j] = (a0 + a1) + (a2 + a3);
}

__global__ void conv_part_final_kernel(const float *__restrict__ P, int splits, TowerGrads ga, TowerGrads gc)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
    if (j >= CONV_PART) return;
    float v = 0.f;
    for (int sidx = 0; sidx < splits; ++sidx) v += P[((size_t)sidx * 2 + t) * CONV_PART + j];
    const TowerGrads &g = t == 0 ? ga : gc;
    if (j < 3072) g.cv2w[j] = v;
    else if (j < 3104) g.cv2b[j - 3072] = v;
    else if (j < 3584) g.cv1w[j - 3104] = v;
    else g.cv1b[j - 3584] = v;
}

// ------------------------------------------------------------------------------------ fp32 GEMM
// C[M,N] = epilogue( sum_k A(m,k) B(k,n) ).  A(m,k) = TA ? A[k*lda+m] : A[m*lda+k];
// B(k,n) = TB ? B[n*ldb+k] : B[k*ldb+n].  Epilogue: + bias[n], ReLU, multiply by (mask[m*ldc+n] > 0).
// 64x64x32 (or 32x64x32) tiles, 256 threads, 4x4 (2x4) micro-tile.  blockIdx.z selects one of up to two independent problems
// (the actor and the critic tower) so both towers share a launch.
struct GemmProblem {
    const float *A, *B, *bias, *mask;
    float *C;
};
struct GemmArgs {
    GemmProblem pr[2];
    int M, N, K, lda, ldb, ldc;
    int relu;
    int ksplit;               // > 1: blockIdx.z = problem * ksplit + split; raw partials to C + split * split_stride
    long long split_stride;
};

constexpr int GEMM_BK = 32;          // k-extent of a tile

template <bool TA, bool TB, int BM>
__global__ void __launch_bounds__(256) gemm_kernel(const GemmArgs g)
{
    constexpr int BK = GEMM_BK, BN = 64, RM = BM / 16;             // RM x 4 micro-tile per thread
    constexpr int NA = BM * BK / 4 / 256, NB = BN * BK / 4 / 256;  // float4 of the A / B tile per thread
    static_assert(BM == 32 || BM == 64, "tile heights");
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int ks = g.ksplit > 1 ? g.ksplit : 1;
    const int prob = blockIdx.z / ks, split = blockIdx.z - prob * ks;
    const GemmProblem pr = prob ? g.pr[1] : g.pr[0];
    const int kper = ((g.K + ks - 1) / ks + 15) / 16 * 16;
    const int kbeg = split * kper, kend = min(g.K, kbeg + kper);
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int tx = tid & 15, ty = tid >> 4;
    float acc[RM][4];
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    // global -> registers (NA float4 of the A tile and NB of the B tile per thread), registers -> shared; the fetch of
    // tile k+1 is issued before the FMAs of tile k so its latency hides behind them.
    auto load4 = [&](const float *src, int i, int lim) {          // src[0..3], elements at index >= lim read as zero
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i + 3 < lim) v = *reinterpret_cast<const float4 *>(src);
        else {
            if (i + 0 < lim) v.x = src[0];
            if (i + 1 < lim) v.y = src[1];
            if (i + 2 < lim) v.z = src[2];
        }
        return v;
    };
    // element (row, k) of a [rows x BK] tile, float4 along k (operand stored row-major along k) or along the rows
    auto fetch_op = [&](bool trans, const float *base, int ld, int r0, int rlim, int rows, int k0, int idx) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!trans) {
            const int r = idx / (BK / 4), kq = (idx % (BK / 4)) * 4;
            const int gr = r0 + r, gk = k0 + kq;
            if (gr < rlim) v = load4(base + (size_t)gr * ld + gk, gk, kend);
        } else {
            const int k = idx / (rows / 4), rq = (idx % (rows / 4)) * 4;
            const int gk = k0 + k, gr = r0 + rq;
            if (gk < kend) v = load4(base + (size_t)gk * ld + gr, gr, rlim);
        }
        return v;
    };
    auto fetch = [&](int k0, float4 (&va)[NA], float4 (&vb)[NB]) {
#pragma unroll
        for (int h = 0; h < NA; ++h) va[h] = fetch_op(TA, pr.A, g.lda, m0, g.M, BM, k0, tid + 256 * h);
#pragma unroll
        for (int h = 0; h < NB; ++h) vb[h] = fetch_op(!TB, pr.B, g.ldb, n0, g.N, BN, k0, tid + 256 * h);
    };
    auto stash = [&](const float4 (&va)[NA], const float4 (&vb)[NB]) {
#pragma unroll
        for (int h = 0; h < NA; ++h) {
            const int idx = tid + 256 * h;
            if (!TA) {
                const int m = idx / (BK / 4), kq = (idx % (BK / 4)) * 4;
                As[kq + 0][m] = va[h].x; As[kq + 1][m] = va[h].y; As[kq + 2][m] = va[h].z; As[kq + 3][m] = va[h].w;
            } else {
                *reinterpret_cast<float4 *>(&As[idx / (BM / 4)][(idx % (BM / 4)) * 4]) = va[h];
            }
        }
#pragma unroll
        for (int h = 0; h < NB; ++h) {
            const int idx = tid + 256 * h;
            if (TB) {
                const int n = idx / (BK / 4), kq = (idx % (BK / 4)) * 4;
                Bs[kq + 0][n] = vb[h].x; Bs[kq + 1][n] = vb[h].y; Bs[kq + 2][n] = vb[h].z; Bs[kq + 3][n] = vb[h].w;
            } else {
                *reinterpret_cast<float4 *>(&Bs[idx / (BN / 4)][(idx % (BN / 4)) * 4]) = vb[h];
            }
        }
    };
    float4 va[NA], vb[NB];
    if (kbeg < kend) fetch(kbeg, va, vb);
    for (int k0 = kbeg; k0 < kend; k0 += BK) {
        stash(va, vb);
        __syncthreads();
        if (k0 + BK < kend) fetch(k0 + BK, va, vb);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float av[RM];
#pragma unroll
            for (int i = 0; i < RM; ++i) av[i] = As[k][ty * RM + i];
            const float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < RM; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < RM; ++i) {
        const int gm = m0 + ty * RM + i;
        if (gm >= g.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int gn = n0 + tx * 4 + j;
            if (gn >= g.N) continue;
            float v = acc[i][j];
            if (ks > 1) { pr.C[(size_t)split * g.split_stride + (size_t)gm * g.ldc + gn] = v; continue; }
            if (pr.bias) v += pr.bias[gn];
            if (g.relu) v = fmaxf(v, 0.0f);
            if (pr.mask) v = pr.mask[(size_t)gm * g.ldc + gn] > 0.0f ? v : 0.0f;
            pr.C[(size_t)gm * g.ldc + gn] = v;
        }
    }
}

// 64-row tiles unless they would leave most SMs without a CTA (the fc2 products at 1024 rows are 64-128 CTAs of 64 rows)
template <bool TA, bool TB>
static void launch_gemm(const GemmArgs &g, int nprob, cudaStream_t s)
{
    const int z = nprob * (g.ksplit > 1 ? g.ksplit : 1);
    const int nx = (g.N + 63) / 64;
    if ((long)nx * ((g.M + 63) / 64) * z < 200) {
        dim3 grid(nx, (g.M + 31) / 32, z);
        gemm_kernel<TA, TB, 32><<<grid, 256, 0, s>>>(g);
    } else {
        dim3 grid(nx, (g.M + 63) / 64, z);
        gemm_kernel<TA, TB, 64><<<grid, 256, 0, s>>>(g);
    }
}

// out_t[j] = sum_s P[(s * 2 + t) * n + j]  (deterministic second stage of every split reduction); grid (ceil(n/256), 2)
__global__ void reduce_splits_kernel(const float *__restrict__ P, int splits, int n, float *out0, float *out1)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
    if (j >= n) return;
    float acc = 0.f;
    for (int sidx = 0; sidx < splits; ++sidx) acc += P[((size_t)sidx * 2 + t) * n + j];
    (t ? out1 : out0)[j] = acc;
}

// ------------------------------------------------------------------------------------ small kernels
// X[t][i][256..259] = goal xy, speed vw for both towers (torch.cat((a, goal, speed)), model/net.py:47,65)
__global__ void fill_gs_kernel(float *__restrict__ X, const float *__restrict__ gs, int nb)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nb) return;
    const float4 v = reinterpret_cast<const float4 *>(gs)[i];
    reinterpret_cast<float4 *>(X + (size_t)i * XLD + 256)[0] = v;
    reinterpret_cast<float4 *>(X + ((size_t)nb + i) * XLD + 256)[0] = v;
}

// heads: one warp per sample.  mean = (sigmoid(actor1), tanh(actor2)), v = critic (model/net.py:49-51,67)
__global__ void heads_fwd_kernel(const float *__restrict__ H2, const float *__restrict__ a1w, const float *__restrict__ a1b,
                                 const float *__restrict__ a2w, const float *__restrict__ a2b,
                                 const float *__restrict__ cw, const float *__restrict__ cb, int nb,
                                 float *__restrict__ value, float *__restrict__ mean)
{
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= nb) return;
    const float4 ha = reinterpret_cast<const float4 *>(H2 + (size_t)i * 128)[lane];
    const float4 hc = reinterpret_cast<const float4 *>(H2 + ((size_t)nb + i) * 128)[lane];
    const float4 w1 = reinterpret_cast<const float4 *>(a1w)[lane], w2 = reinterpret_cast<const float4 *>(a2w)[lane],
                 w3 = reinterpret_cast<const float4 *>(cw)[lane];
    float z1 = fmaf(ha.x, w1.x, fmaf(ha.y, w1.y, fmaf(ha.z, w1.z, ha.w * w1.w)));
    float z2 = fmaf(ha.x, w2.x, fmaf(ha.y, w2.y, fmaf(ha.z, w2.z, ha.w * w2.w)));
    float z3 = fmaf(hc.x, w3.x, fmaf(hc.y, w3.y, fmaf(hc.z, w3.z, hc.w * w3.w)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        z1 += __shfl_xor_sync(0xffffffffu, z1, o);
        z2 += __shfl_xor_sync(0xffffffffu, z2, o);
        z3 += __shfl_xor_sync(0xffffffffu, z3, o);
    }
    if (lane == 0) {
        z1 += a1b[0]; z2 += a2b[0]; z3 += cb[0];
        mean[2 * i + 0] = 1.0f / (1.0f + expf(-z1));
        mean[2 * i + 1] = tanhf(z2);
        value[i] = z3;
    }
}

#define HEAD_CHUNK 8
// dZ2[t][i][j] for both towers + per-chunk partial sums of the three head weight/bias gradients.
// block = 128 threads (one per hidden unit j), grid = chunks of HEAD_CHUNK samples.
__global__ void __launch_bounds__(128) heads_bwd_kernel(const float *__restrict__ H2, const float *__restrict__ dOut,
                                                        const float *__restrict__ a1w, const float *__restrict__ a2w,
                                                        const float *__restrict__ cw, int nb, float *__restrict__ dZ2,
                                                        float *__restrict__ headpart)
{
    const int j = threadIdx.x, c = blockIdx.x;
    const float w1 = a1w[j], w2 = a2w[j], w3 = cw[j];
    float g1 = 0.f, g2 = 0.f, g3 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
    const int i1 = min(nb, (c + 1) * HEAD_CHUNK);
    for (int i = c * HEAD_CHUNK; i < i1; ++i) {
        const float4 d = reinterpret_cast<const float4 *>(dOut)[i];     // dv, dz1, dz2, _
        const float ha = H2[(size_t)i * 128 + j], hc = H2[((size_t)nb + i) * 128 + j];
        dZ2[(size_t)i * 128 + j] = ha > 0.0f ? fmaf(d.y, w1, d.z * w2) : 0.0f;
        dZ2[((size_t)nb + i) * 128 + j] = hc > 0.0f ? d.x * w3 : 0.0f;
        g1 = fmaf(d.y, ha, g1); g2 = fmaf(d.z, ha, g2); g3 = fmaf(d.x, hc, g3);
        b1 += d.y; b2 += d.z; b3 += d.x;
    }
    float *o = headpart + (size_t)c * 3 * 132;
    o[0 * 132 + j] = g1; o[1 * 132 + j] = g2; o[2 * 132 + j] = g3;
    if (j == 0) { o[0 * 132 + 128] = b1; o[1 * 132 + 128] = b2; o[2 * 132 + 128] = b3; }
}

#define HPR_GROUPS 7      // 7 x 132 = 924 threads: each group sums every 7th chunk, fixed-order combine (deterministic)
__global__ void __launch_bounds__(HPR_GROUPS * 132)
heads_part_reduce_kernel(const float *__restrict__ headpart, int chunks, float *ga1w, float *ga1b, float *ga2w,
                         float *ga2b, float *gcw, float *gcb)
{
    __shared__ float red[HPR_GROUPS][132];
    const int g = threadIdx.x / 132, j = threadIdx.x - g * 132, h = blockIdx.x;     // 3 blocks: actor1, actor2, critic
    float acc = 0.f;
    if (j <= 128)
        for (int c = g; c < chunks; c += HPR_GROUPS) acc += headpart[((size_t)c * 3 + h) * 132 + j];
    red[g][j] = acc;
    __syncthreads();
    if (g == 0 && j <= 128) {
#pragma unroll
        for (int k = 1; k < HPR_GROUPS; ++k) acc += red[k][j];
        float *w = h == 0 ? ga1w : (h == 1 ? ga2w : gcw), *b = h == 0 ? ga1b : (h == 1 ? ga2b : gcb);
        if (j < 128) w[j] = acc; else b[0] = acc;
    }
}

// out[t][j] = sum_i A[t][i*ld + j] ; grid (ceil(ncols/32), ntowers), 256 threads = 8 row groups x 32 columns
struct ColsumArgs { const float *A[2]; float *P; int rows, cols, ld; };
__global__ void __launch_bounds__(256) colsum_kernel(const ColsumArgs a)
{
    __shared__ float red[8][33];
    const int t = blockIdx.y, lane = threadIdx.x & 31, rg = threadIdx.x >> 5;
    const int j = blockIdx.x * 32 + lane;
    float acc = 0.f;
    const int rper = (a.rows + gridDim.z - 1) / gridDim.z;
    const int r0 = blockIdx.z * rper, r1 = min(a.rows, r0 + rper);
    if (j < a.cols)
        {
        const float *A = t ? a.A[1] : a.A[0];
        for (int i = r0 + rg; i < r1; i += 8) acc += A[(size_t)i * a.ld + j];
    }
    red[rg][lane] = acc;
    __syncthreads();
    if (rg == 0 && j < a.cols) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < 8; ++r) s += red[r][lane];
        a.P[((size_t)blockIdx.z * 2 + t) * a.cols + j] = s;
    }
}

// ------------------------------------------------------------------------------------ sampling
__device__ __forceinline__ void philox4(uint32_t (&c)[4], uint32_t k0, uint32_t k1)
{
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
        uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
        uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}

#define LOG_2PI_HALF 0.91893853320467274178f

__global__ void sample_kernel(const float *__restrict__ logstd, const float *__restrict__ mean, int nb, uint64_t seed,
                              uint64_t counter, int deterministic, float *__restrict__ action,
                              float *__restrict__ logprob, float *__restrict__ scaled)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nb) return;
    const float ls0 = logstd[0], ls1 = logstd[1];
    const float m0 = mean[2 * i], m1 = mean[2 * i + 1];
    float a0 = m0, a1 = m1;
    if (deterministic == 2) { a0 = action[2 * i]; a1 = action[2 * i + 1]; }   // evaluate a given action
    if (!deterministic) {
        uint32_t c[4] = {(uint32_t)i, (uint32_t)counter, (uint32_t)(counter >> 32), 0x5A17u};
        philox4(c, (uint32_t)seed, (uint32_t)(seed >> 32));
        // Box-Muller on two 24-bit uniforms in (0,1]
        const float u1 = ((float)(c[0] >> 8) + 1.0f) * 5.9604644775390625e-08f;
        const float u2 = (float)(c[1] >> 8) * 5.9604644775390625e-08f;
        const float rad = sqrtf(-2.0f * logf(u1));
        float sn, cs;
        sincosf(6.28318530717958647692f * u2, &sn, &cs);
        a0 = fmaf(expf(ls0), rad * cs, m0);
        a1 = fmaf(expf(ls1), rad * sn, m1);
    }
    // log_normal_density (model/utils.py:90-97)
    const float d0 = a0 - m0, d1 = a1 - m1;
    const float v0 = expf(2.0f * ls0), v1 = expf(2.0f * ls1);
    const float lp = (-(d0 * d0) / (2.0f * v0) - LOG_2PI_HALF - ls0) + (-(d1 * d1) / (2.0f * v1) - LOG_2PI_HALF - ls1);
    action[2 * i] = a0; action[2 * i + 1] = a1;
    logprob[i] = lp;
    if (scaled) {
        scaled[2 * i] = fminf(fmaxf(a0, 0.0f), 1.0f);          // action_bound [[0,-1],[1,1]] (ppo_stage1.py:170)
        scaled[2 * i + 1] = fminf(fmaxf(a1, -1.0f), 1.0f);
    }
}

// ------------------------------------------------------------------------------------ PPO loss (+ gradient)
// single CTA of 1024 threads; deterministic tree reductions.
__device__ __forceinline__ float block_sum_1024(float v, float *sh)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = (threadIdx.x < 32) ? sh[threadIdx.x] : 0.0f;
    if (threadIdx.x < 32) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
        if (threadIdx.x == 0) sh[32] = r;
    }
    __syncthreads();
    return sh[32];
}

__global__ void __launch_bounds__(1024) ppo_loss_kernel(const float *__restrict__ logstd, const float *__restrict__ value,
                                                        const float *__restrict__ mean, const float *__restrict__ action,
                                                        const float *__restrict__ old_lp, const float *__restrict__ adv,
                                                        const float *__restrict__ target, int nb, float clip,
                                                        float coeff_entropy, float value_coef, float weight,
                                                        float *__restrict__ dOut, float *__restrict__ losses,
                                                        float *__restrict__ dlogstd)
{
    __shared__ float sh[34];
    const float ls0 = logstd[0], ls1 = logstd[1];
    const float var0 = expf(2.0f * ls0), var1 = expf(2.0f * ls1);
    const float inv_nb = 1.0f / (float)nb;
    const float ginv = weight * inv_nb;          // gradients carry the data-parallel row weight, the logged losses do not
    float s_pl = 0.f, s_vl = 0.f, s_g0 = 0.f, s_g1 = 0.f;
    for (int i = threadIdx.x; i < nb; i += 1024) {
        const float m0 = mean[2 * i], m1 = mean[2 * i + 1];
        const float d0 = action[2 * i] - m0, d1 = action[2 * i + 1] - m1;
        const float lp = (-(d0 * d0) / (2.0f * var0) - LOG_2PI_HALF - ls0) + (-(d1 * d1) / (2.0f * var1) - LOG_2PI_HALF - ls1);
        const float ratio = expf(lp - old_lp[i]);
        const float A = adv[i];
        const float s1 = ratio * A;
        const float s2 = fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip) * A;
        s_pl += fminf(s1, s2);
        const float dv = value[i] - target[i];
        s_vl += dv * dv;
        // d(-mean(min))/d lp : gradient flows through s1 when s1 <= s2 (ties split evenly in torch and both
        // halves reach `ratio`), else through the clamp, which is flat outside its range.
        const float g_lp = (s1 <= s2) ? -ginv * A * ratio : 0.0f;
        const float dm0 = g_lp * d0 / var0, dm1 = g_lp * d1 / var1;      // dL/dmean
        s_g0 += g_lp * (d0 * d0 / var0 - 1.0f);
        s_g1 += g_lp * (d1 * d1 / var1 - 1.0f);
        reinterpret_cast<float4 *>(dOut)[i] =
            make_float4(value_coef * 2.0f * dv * ginv, dm0 * m0 * (1.0f - m0), dm1 * (1.0f - m1 * m1), 0.0f);
    }
    const float pl = block_sum_1024(s_pl, sh), vl = block_sum_1024(s_vl, sh);
    const float g0 = block_sum_1024(s_g0, sh), g1 = block_sum_1024(s_g1, sh);
    if (threadIdx.x == 0) {
        losses[0] = -pl * inv_nb;                              // policy_loss
        losses[1] = vl * inv_nb;                               // value_loss
        losses[2] = (0.5f + LOG_2PI_HALF + ls0) + (0.5f + LOG_2PI_HALF + ls1);   // dist_entropy (model/net.py:78-79)
        dlogstd[0] = g0 - coeff_entropy * weight;
        dlogstd[1] = g1 - coeff_entropy * weight;
    }
}

// ------------------------------------------------------------------------------------ behaviour-cloning loss (+ gradient)
// loss = mean_i sum_k (mean_ik - a_ik)^2 on the deterministic action; single CTA of 1024 threads, deterministic tree
// reduction.  Only the actor heads get a gradient: dv = 0, so the critic tower's gradients are exactly zero, and the
// logstd gradient (pol->red) is 0.
__global__ void __launch_bounds__(1024) bc_loss_kernel(const float *__restrict__ mean, const float *__restrict__ target,
                                                       int nb, float *__restrict__ dOut, float *__restrict__ loss,
                                                       float *__restrict__ dlogstd)
{
    __shared__ float sh[34];
    const float inv_nb = 1.0f / (float)nb;
    float s = 0.f;
    for (int i = threadIdx.x; i < nb; i += 1024) {
        const float m0 = mean[2 * i], m1 = mean[2 * i + 1];
        const float e0 = m0 - target[2 * i], e1 = m1 - target[2 * i + 1];
        s += e0 * e0 + e1 * e1;
        const float g0 = 2.0f * inv_nb * e0, g1 = 2.0f * inv_nb * e1;                  // dL/dmean
        reinterpret_cast<float4 *>(dOut)[i] = make_float4(0.0f, g0 * m0 * (1.0f - m0), g1 * (1.0f - m1 * m1), 0.0f);
    }
    const float tot = block_sum_1024(s, sh);
    if (threadIdx.x == 0) {
        loss[0] = tot * inv_nb;
        dlogstd[0] = 0.0f;
        dlogstd[1] = 0.0f;
    }
}

// ------------------------------------------------------------------------------------ Adam / GAE / misc
__global__ void adam_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                            float *__restrict__ v, int64_t n, float lr, float b1, float b2, float eps, float bc1,
                            float bc2_sqrt, float grad_scale)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float gi = g[i] * grad_scale;
    const float mi = fmaf(b1, m[i], (1.0f - b1) * gi);
    const float vi = fmaf(b2, v[i], (1.0f - b2) * gi * gi);
    m[i] = mi; v[i] = vi;
    // torch.optim.Adam: denom = sqrt(v)/sqrt(bias_correction2) + eps ; p -= lr/bias_correction1 * m/denom
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] -= (lr / bc1) * (mi / denom);
}

// The optimizer step of a policy workspace: Adam over the whole flat buffer AND the tf32 hi / lo split of the two fc1
// weight matrices (97 % of the parameters) with their transposes, which the next forward / backward GEMMs read - the
// split would otherwise be a pass of its own at the head of every forward after a step, on the critical path.
// Blocks below tile_blocks take a 32 x 32 tile of fc1w[tower] (coalesced rows in, coalesced rows out, the transposed
// copies through a padded shared tile, as split_both_kernel); the others take the parameters outside those ranges
// element-wise.  The arithmetic is adam_kernel's, expression for expression.
struct AdamSplitArgs {
    float *p, *m, *v;
    const float *g;
    long long n, w_off0, w_off1;
    float *hi0, *lo0, *thi0, *tlo0, *hi1, *lo1, *thi1, *tlo1;
    float lr, b1, b2, eps, bc1, bc2_sqrt, grad_scale;
    int tile_blocks;
};

__device__ __forceinline__ float adam_update_one(const AdamSplitArgs &a, long long i)
{
    const float gi = a.g[i] * a.grad_scale;
    const float mi = fmaf(a.b1, a.m[i], (1.0f - a.b1) * gi);
    const float vi = fmaf(a.b2, a.v[i], (1.0f - a.b2) * gi * gi);
    a.m[i] = mi; a.v[i] = vi;
    const float denom = sqrtf(vi) / a.bc2_sqrt + a.eps;
    float pv = a.p[i];
    pv -= (a.lr / a.bc1) * (mi / denom);
    a.p[i] = pv;
    return pv;
}

__global__ void __launch_bounds__(256) adam_split_kernel(const AdamSplitArgs a)
{
    __shared__ float tile[32][33];
    constexpr long long WSZ = 256LL * FEAT;
    if ((int)blockIdx.x < a.tile_blocks) {
        const int t = blockIdx.x >> 10, rem = blockIdx.x & 1023;       // 8 x 128 tiles per tower
        const int r0 = (rem >> 7) * 32, c0 = (rem & 127) * 32;
        const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
        const long long base = t ? a.w_off1 : a.w_off0;
        float *hi = t ? a.hi1 : a.hi0, *lo = t ? a.lo1 : a.lo0, *thi = t ? a.thi1 : a.thi0, *tlo = t ? a.tlo1 : a.tlo0;
        for (int i = ty; i < 32; i += 8) {
            const long long e = (long long)(r0 + i) * FEAT + c0 + tx;
            const float x = adam_update_one(a, base + e);
            const float h = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
            hi[e] = h;
            lo[e] = x - h;
            tile[i][tx] = x;
        }
        __syncthreads();
        for (int i = ty; i < 32; i += 8) {
            const float x = tile[tx][i];
            const float h = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
            const long long e = (long long)(c0 + i) * 256 + r0 + tx;
            thi[e] = h;
            tlo[e] = x - h;
        }
    } else {
        long long i = (long long)(blockIdx.x - a.tile_blocks) * 256 + threadIdx.x;
        if (i >= a.w_off0) i += WSZ;               // skip the two fc1w ranges
        if (i >= a.w_off1) i += WSZ;
        if (i < a.n) adam_update_one(a, i);
    }
}

// GAE as a blocked segmented scan over time (generate_train_data, model/ppo.py:122-139).
// The recurrence A_t = delta_t + k_t A_{t+1} (k_t = gamma*lam*(1-d_t); a done flag cuts the segment) is affine, so a
// chunk of GAE_CHUNK steps composes to A_first = P + Q * A_after.  Block = 8 time chunks x 32 agents:
//   pass 1: every (chunk, agent) thread folds its chunk into (P, Q);        [parallel over T/GAE_CHUNK chunks]
//   pass 2: the carry entering each chunk is folded from the later chunks in shared memory;
//   pass 3: every thread replays its chunk from the carry and writes targets / advantages.
// float64 like the reference's numpy; inputs are time-major (T, N) so a warp reads 32 consecutive agents (coalesced).
#define GAE_CHUNKS 8
__global__ void __launch_bounds__(256) gae_kernel(const float *__restrict__ rewards, const float *__restrict__ values,
                                                  const float *__restrict__ last_value, const uint8_t *__restrict__ dones,
                                                  int T, int N, double gamma, double lam, float *__restrict__ targets,
                                                  float *__restrict__ advs)
{
    __shared__ double sP[GAE_CHUNKS][32], sQ[GAE_CHUNKS][32];
    const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + lane;
    const int clen = (T + GAE_CHUNKS - 1) / GAE_CHUNKS;
    const int t0 = c * clen, t1 = min(T, t0 + clen);            // this thread's time range [t0, t1)
    const bool act = i < N;
    double P = 0.0, Q = 1.0;
    if (act) {
        for (int t = t1 - 1; t >= t0; --t) {
            const size_t k = (size_t)t * N + i;
            const double nd = dones[k] ? 0.0 : 1.0;
            const double vnext = (t + 1 < T) ? (double)values[k + N] : (double)last_value[i];
            const double delta = (double)rewards[k] + gamma * vnext * nd - (double)values[k];
            const double kk = gamma * lam * nd;
            // A_t = delta + kk * (P + Q * A_after)
            P = delta + kk * P;
            Q = kk * Q;
        }
    }
    sP[c][lane] = P; sQ[c][lane] = Q;
    __syncthreads();
    double carry = 0.0;                                          // A just after this chunk
    for (int cc = GAE_CHUNKS - 1; cc > c; --cc) carry = sP[cc][lane] + sQ[cc][lane] * carry;
    if (act) {
        double gae = carry;
        for (int t = t1 - 1; t >= t0; --t) {
            const size_t k = (size_t)t * N + i;
            const double nd = dones[k] ? 0.0 : 1.0;
            const double v = (double)values[k];
            const double vnext = (t + 1 < T) ? (double)values[k + N] : (double)last_value[i];
            const double delta = (double)rewards[k] + gamma * vnext * nd - v;
            gae = delta + gamma * lam * nd * gae;
            const double tgt = gae + v;
            targets[k] = (float)tgt;
            advs[k] = (float)(tgt - v);
        }
    }
}

__global__ void obs_stack_push_kernel(const float4 *__restrict__ in, const float4 *__restrict__ obs,
                                      const uint8_t *__restrict__ flags, int n, int b4, float4 *__restrict__ out)
{
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)n * b4) return;
    const int a = (int)(idx / b4), j = (int)(idx - (int64_t)a * b4);
    const float4 o = obs[idx];
    const bool was_reset = flags != nullptr && flags[4 * a + 3] != 0;
    const size_t base = (size_t)a * 3 * b4 + j;
    out[base] = was_reset ? o : in[base + b4];
    out[base + b4] = was_reset ? o : in[base + 2 * (size_t)b4];
    out[base + 2 * (size_t)b4] = o;
}

// advs = (advs - mean) / std over the whole rollout, numpy semantics (ddof = 0, float64 moments, no epsilon):
// model/ppo.py:148.  Single CTA; `moments` (3 doubles: sum, sum of squares, count) lets a data-parallel
// caller all-reduce the moments between the two phases.
__global__ void __launch_bounds__(1024) adv_moments_kernel(const float *__restrict__ x, int64_t n, double *moments)
{
    __shared__ double sh[2][32];
    double s = 0.0, ss = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += 1024) { const double v = (double)x[i]; s += v; ss += v * v; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ss += __shfl_xor_sync(0xffffffffu, ss, o); }
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s; sh[1][threadIdx.x >> 5] = ss; }
    __syncthreads();
    if (threadIdx.x < 32) {
        s = sh[0][threadIdx.x]; ss = sh[1][threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ss += __shfl_xor_sync(0xffffffffu, ss, o); }
        if (threadIdx.x == 0) { moments[0] = s; moments[1] = ss; moments[2] = (double)n; }
    }
}

__global__ void adv_apply_kernel(const float *__restrict__ x, int64_t n, const double *__restrict__ moments,
                                 float *__restrict__ out)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double cnt = moments[2], mean = moments[0] / cnt;
    const double var = moments[1] / cnt - mean * mean;
    out[i] = (float)(((double)x[i] - mean) / sqrt(var));
}

// dst[i, :] = src[idx[i], :] for rows of row_floats floats (multiple of 4): minibatch assembly (model/ppo.py:162-169)
__global__ void gather_rows_kernel(const float4 *__restrict__ src, const int64_t *__restrict__ idx, int row4, int nrows,
                                   float4 *__restrict__ dst)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)nrows * row4) return;
    const int r = (int)(t / row4), j = (int)(t - (int64_t)r * row4);
    dst[t] = src[idx[r] * row4 + j];
}

__global__ void gather_scalar_kernel(const float *__restrict__ src, const int64_t *__restrict__ idx, int row, int nrows,
                                     float *__restrict__ dst)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nrows * row) return;
    const int r = t / row, j = t - r * row;
    dst[t] = src[idx[r] * row + j];
}

// The six arrays of one PPO minibatch (observation stack, goal | speed, action, log-prob, advantage, target:
// model/ppo.py:162-169) gathered by the same index in ONE launch: blockIdx.y = array, blockIdx.x covers the largest.
struct GatherMulti {
    const float *src[RLCA_GATHER_MAX];
    float *dst[RLCA_GATHER_MAX];
    int row[RLCA_GATHER_MAX];
};

__global__ void gather_multi_kernel(const GatherMulti g, const int64_t *__restrict__ idx, int nrows)
{
    const int a = blockIdx.y;
    const int row = g.row[a];
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if ((row & 3) == 0) {
        const int row4 = row >> 2;
        if (t >= (int64_t)nrows * row4) return;
        const int r = (int)(t / row4), j = (int)(t - (int64_t)r * row4);
        reinterpret_cast<float4 *>(g.dst[a])[t] = reinterpret_cast<const float4 *>(g.src[a])[idx[r] * row4 + j];
    } else {
        if (t >= (int64_t)nrows * row) return;
        const int r = (int)(t / row), j = (int)(t - (int64_t)r * row);
        g.dst[a][t] = g.src[a][idx[r] * row + j];
    }
}

// ------------------------------------------------------------------------------------ host API
extern "C" int rlca_adv_moments(const float *x, int64_t n, double *moments, void *stream)
{
    if (!x || !moments || n < 1) return rlca_set_err(RLCA_ERR_INVALID, "bad adv_moments arguments");
    adv_moments_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(x, n, moments);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_adv_apply(const float *x, int64_t n, const double *moments, float *out, void *stream)
{
    if (!x || !moments || !out || n < 1) return rlca_set_err(RLCA_ERR_INVALID, "bad adv_apply arguments");
    adv_apply_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, n, moments, out);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_gather_rows(const float *src, const int64_t *idx, int32_t row_floats, int32_t nrows, float *dst,
                                void *stream)
{
    if (!src || !idx || !dst || row_floats < 1 || nrows < 1) return rlca_set_err(RLCA_ERR_INVALID, "bad gather arguments");
    if ((row_floats & 3) == 0) {
        const int row4 = row_floats / 4;
        const int64_t total = (int64_t)nrows * row4;
        gather_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
            reinterpret_cast<const float4 *>(src), idx, row4, nrows, reinterpret_cast<float4 *>(dst));
    } else {
        const int total = nrows * row_floats;
        gather_scalar_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(src, idx, row_floats, nrows, dst);
    }
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_gather_minibatch(const float *const *src, const int32_t *row_floats, int32_t narrays,
                                     const int64_t *idx, int32_t nrows, float *const *dst, void *stream)
{
    if (!src || !row_floats || !idx || !dst || narrays < 1 || narrays > RLCA_GATHER_MAX || nrows < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "bad gather_minibatch arguments");
    GatherMulti g{};
    int64_t most = 0;
    for (int a = 0; a < narrays; ++a) {
        if (!src[a] || !dst[a] || row_floats[a] < 1) return rlca_set_err(RLCA_ERR_INVALID, "bad gather_minibatch array");
        // the float4 path needs 16-byte aligned rows on both sides
        const bool vec = (row_floats[a] & 3) == 0 && (((uintptr_t)src[a] | (uintptr_t)dst[a]) & 15) == 0;
        g.src[a] = src[a]; g.dst[a] = dst[a];
        g.row[a] = row_floats[a];
        if (!vec && (row_floats[a] & 3) == 0) return rlca_set_err(RLCA_ERR_INVALID, "gather_minibatch: rows of 4k floats must be 16-byte aligned");
        const int64_t units = (int64_t)nrows * (vec ? row_floats[a] / 4 : row_floats[a]);
        if (units > most) most = units;
    }
    gather_multi_kernel<<<dim3((unsigned)((most + 255) / 256), narrays), 256, 0, (cudaStream_t)stream>>>(g, idx, nrows);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_policy_create(int32_t max_batch, rlca_policy **out)
{
    if (!out || max_batch < 1) return rlca_set_err(RLCA_ERR_INVALID, "bad max_batch/out");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return rlca_set_err(RLCA_ERR_NO_DEVICE, "no CUDA device; librlca has no CPU fallback");
    rlca_policy *p = new (std::nothrow) rlca_policy();
    if (!p) return rlca_set_err(RLCA_ERR_INVALID, "out of host memory");
    memset(p, 0, sizeof(*p));
    p->max_batch = max_batch;
    const size_t B = (size_t)max_batch;
    const int chunks = (max_batch + HEAD_CHUNK - 1) / HEAD_CHUNK;
    RLCA_CUDA_TRY(cudaMalloc(&p->F, 2 * B * FEAT * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->X, 2 * B * XLD * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->H2, 2 * B * 128 * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->dOut, B * 4 * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->dZ2, 2 * B * 128 * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->dX, 2 * B * XLD * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->dF, 2 * B * FEAT * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->part, 2 * (B > 128 ? B : 128) * CONV_PART * sizeof(float)));   // >= one slot per CTA of the tc backward
    RLCA_CUDA_TRY(cudaMalloc(&p->headpart, (size_t)chunks * 3 * 132 * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->red, 64 * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->Wc, 2 * CONV_WBLK * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->S, (size_t)RSPLIT * 2 * 128 * XLD * sizeof(float)));
    RLCA_CUDA_TRY(cudaMalloc(&p->S2, (size_t)RSPLIT * 2 * CONV_PART * sizeof(float)));
    for (int i = 0; i < 2; ++i) {
        RLCA_CUDA_TRY(cudaStreamCreateWithFlags(&p->side[i], cudaStreamNonBlocking));
        RLCA_CUDA_TRY(cudaEventCreateWithFlags(&p->ev_join[i], cudaEventDisableTiming));
    }
    RLCA_CUDA_TRY(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
    RLCA_CUDA_TRY(cudaEventCreateWithFlags(&p->ev_heads, cudaEventDisableTiming));
    RLCA_CUDA_TRY(cudaEventCreateWithFlags(&p->ev_dx, cudaEventDisableTiming));
    RLCA_CUDA_TRY(cudaEventCreateWithFlags(&p->ev_split, cudaEventDisableTiming));
    RLCA_CUDA_TRY(cudaEventCreateWithFlags(&p->ev_prep, cudaEventDisableTiming));
    {
        const char *e = getenv("RLCA_BWD_STREAMS");          // read once, at creation
        p->use_side = !(e && atoi(e) == 0);
    }
    p->bpad = (max_batch + 31) / 32 * 32;
    {
        const size_t BP = (size_t)p->bpad;
        RLCA_CUDA_TRY(cudaMalloc(&p->Fs, 4 * B * FEAT * sizeof(float)));
        RLCA_CUDA_TRY(cudaMalloc(&p->W1s, 4 * (size_t)256 * FEAT * sizeof(float)));
        RLCA_CUDA_TRY(cudaMalloc(&p->W1Ts, 4 * (size_t)256 * FEAT * sizeof(float)));
        RLCA_CUDA_TRY(cudaMalloc(&p->dZs, 4 * B * 256 * sizeof(float)));
        RLCA_CUDA_TRY(cudaMalloc(&p->dZTs, 4 * 256 * BP * sizeof(float)));
        RLCA_CUDA_TRY(cudaMalloc(&p->FTs, 4 * (size_t)FEAT * BP * sizeof(float)));
        RLCA_CUDA_TRY(cudaMalloc(&p->P, 8 * 2 * B * 256 * sizeof(float)));
        int rc = rlca_tc_init();
        if (rc) return rc;
        p->use_tc = 1;
        p->weights_dirty = 1;
        p->wimg_dirty = 1;
        p->wc_dirty = 1;
        rc = rlca_conv_tc_init();
        if (rc) return rc;
        RLCA_CUDA_TRY(cudaMalloc(&p->Wimg, rlca_conv_tc_image_floats() * sizeof(float)));
        RLCA_CUDA_TRY(cudaMalloc(&p->WimgB, rlca_conv_tc_bwd_image_floats() * sizeof(float)));
        p->conv_bwd_dirty = 1;
        int dev = 0;
        RLCA_CUDA_TRY(cudaGetDevice(&dev));
        RLCA_CUDA_TRY(cudaDeviceGetAttribute(&p->num_sms, cudaDevAttrMultiProcessorCount, dev));
        p->use_tc_conv = 1;
    }
    RLCA_CUDA_TRY(cudaFuncSetAttribute(conv_tower_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)sizeof(ConvSmem)));
    RLCA_CUDA_TRY(cudaFuncSetAttribute(conv_tower_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)sizeof(ConvBwdSmem)));
    *out = p;
    return RLCA_OK;
}

extern "C" int rlca_policy_destroy(rlca_policy *p)
{
    if (!p) return RLCA_OK;
    cudaFree(p->F); cudaFree(p->X); cudaFree(p->H2); cudaFree(p->dOut); cudaFree(p->dZ2); cudaFree(p->dX);
    cudaFree(p->dF); cudaFree(p->part); cudaFree(p->headpart); cudaFree(p->red); cudaFree(p->S); cudaFree(p->Wc);
    cudaFree(p->S2);
    for (int i = 0; i < 2; ++i) { if (p->side[i]) cudaStreamDestroy(p->side[i]); if (p->ev_join[i]) cudaEventDestroy(p->ev_join[i]); }
    if (p->ev_fork) cudaEventDestroy(p->ev_fork);
    if (p->ev_heads) cudaEventDestroy(p->ev_heads);
    if (p->ev_dx) cudaEventDestroy(p->ev_dx);
    if (p->ev_split) cudaEventDestroy(p->ev_split);
    if (p->ev_prep) cudaEventDestroy(p->ev_prep);
    cudaFree(p->Fs); cudaFree(p->W1s); cudaFree(p->W1Ts); cudaFree(p->dZs); cudaFree(p->dZTs); cudaFree(p->FTs); cudaFree(p->P); cudaFree(p->Wimg); cudaFree(p->WimgB);
    delete p;
    return RLCA_OK;
}

extern "C" int64_t rlca_policy_launch_count(const rlca_policy *p) { return p ? p->launches : -1; }

extern "C" int rlca_policy_set_grad_event(rlca_policy *pol, void *event)
{
    if (!pol) return rlca_set_err(RLCA_ERR_INVALID, "NULL workspace");
    pol->fc_grads_event = (cudaEvent_t)event;
    // The conv tower backward is a persistent kernel whose CTAs fill every SM's shared memory: an NCCL kernel launched
    // meanwhile would only start when it ends.  While a gradient event is set it runs on 16 SMs fewer, so that the
    // all-reduce can run under the dF GEMM + conv backward instead of following them.
    pol->reserved_sms = event ? 16 : 0;
    if (event) { const char *e = getenv("RLCA_RESERVED_SMS"); if (e) pol->reserved_sms = atoi(e); }     // experiment knob
    return RLCA_OK;
}

extern "C" int rlca_policy_weights_changed(rlca_policy *p)
{
    if (!p) return rlca_set_err(RLCA_ERR_INVALID, "policy is NULL");
    p->weights_dirty = 1;
    p->wimg_dirty = 1;
    p->conv_bwd_dirty = 1;
    p->wc_dirty = 1;
    p->w1_split_valid = 0;
    return RLCA_OK;
}

extern "C" int rlca_policy_set_tensor_cores(rlca_policy *p, int32_t enable)
{
    if (!p) return rlca_set_err(RLCA_ERR_INVALID, "policy is NULL");
    p->use_tc = enable ? 1 : 0;
    p->use_tc_conv = enable == 1 ? 1 : 0;      // 2 = fc1 GEMMs only (conv tower on the CUDA cores)
    p->weights_dirty = 1;
    p->wimg_dirty = 1;
    p->conv_bwd_dirty = 1;
    p->wc_dirty = 1;
    p->w1_split_valid = 0;
    return RLCA_OK;
}

extern "C" int rlca_policy_features(const rlca_policy *pol, int32_t tower, int32_t nb, float *dst_dev, void *stream)
{
    if (!pol || !dst_dev || tower < 0 || tower > 1 || nb < 1 || nb > pol->max_batch)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_policy_features: bad argument");
    // F is [2][nb of the last forward][4096]; the caller passes the same nb
    RLCA_CUDA_TRY(cudaMemcpyAsync(dst_dev, pol->F + (size_t)tower * nb * FEAT, (size_t)nb * FEAT * sizeof(float),
                                  cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return RLCA_OK;
}

extern "C" int rlca_policy_forward(rlca_policy *pol, const float *params, const float *obs, const float *gs, int32_t nb,
                                   float *value, float *mean, void *stream)
{
    if (!pol || !params || !obs || !gs || !value || !mean) return rlca_set_err(RLCA_ERR_INVALID, "NULL argument");
    if (nb < 1 || nb > pol->max_batch) return rlca_set_err(RLCA_ERR_INVALID, "nb exceeds the workspace max_batch");
    cudaStream_t s = (cudaStream_t)stream;
    const TowerPtrs ta = tower_ptrs(params, 0), tc = tower_ptrs(params, 1);
    // the tensor-core conv tower stages the scan with 16-byte bulk copies; oddly aligned inputs take the CUDA-core kernel
    // (which leaves Wimg as it is: its own dirty flag keeps it stale until the next forward that reads it)
    if (pol->use_tc && pol->use_tc_conv && ((uintptr_t)obs & 15) == 0) {
        if (pol->wimg_dirty) {
            const float *w1[2] = {ta.cv1w, tc.cv1w}, *b1[2] = {ta.cv1b, tc.cv1b};
            const float *w2[2] = {ta.cv2w, tc.cv2w}, *b2[2] = {ta.cv2b, tc.cv2b};
            rlca_conv_tc_prep(w1, b1, w2, b2, pol->Wimg, s);
            pol->wimg_dirty = 0;
            pol->launches += 1;
        }
        int rc = rlca_conv_tc_forward(obs, pol->Wimg, pol->F, pol->Fs, nb, pol->num_sms, s);
        if (rc) return rc;
    } else {
        if (pol->wc_dirty) {
            conv_prep_weights_kernel<<<dim3((CONV_WBLK + 255) / 256, 2), 256, 0, s>>>(ta, tc, pol->Wc);
            pol->wc_dirty = 0;
            pol->launches += 1;
        }
        conv_tower_fwd_kernel<<<(nb + CONV_SPC - 1) / CONV_SPC, 256, sizeof(ConvSmem), s>>>(
            obs, pol->Wc, pol->F, pol->use_tc ? pol->Fs : nullptr, nb);
    }
    GemmArgs g{};
    if (pol->use_tc) {
        // fc1 on the tensor cores: split F and W1 into tf32 hi/lo parts, split-K 3xTF32 GEMM, fused bias+ReLU reduce
        const size_t B = (size_t)nb;
        const size_t WSZ = (size_t)256 * FEAT;
        RlcaTcProblem pr[2];
        for (int t = 0; t < 2; ++t) {
            float *Fh = pol->Fs + (size_t)(2 * t) * B * FEAT, *Fl = Fh + B * FEAT;
            float *Wh = pol->W1s + (size_t)(2 * t) * WSZ, *Wl = Wh + WSZ;
            pr[t] = RlcaTcProblem{Fh, Fl, Wh, Wl, FEAT, FEAT, pol->P + (size_t)t * B * 256, nullptr};
        }
        if (pol->weights_dirty && !pol->w1_split_valid) {   // hi/lo (and transposed) copies of W1 after a weight change the optimizer step did not make
            const float *w[2] = {ta.fc1w, tc.fc1w};
            float *hi[2], *lo[2], *thi[2], *tlo[2];
            for (int t = 0; t < 2; ++t) {
                hi[t] = pol->W1s + (size_t)(2 * t) * WSZ; lo[t] = hi[t] + WSZ;
                thi[t] = pol->W1Ts + (size_t)(2 * t) * WSZ; tlo[t] = thi[t] + WSZ;
            }
            rlca_tc_split_both(w, 256, FEAT, FEAT, hi, lo, FEAT, thi, tlo, 256, s);
        }
        const int mtiles = (nb + 127) / 128;
        int splits = 1;
        while (splits < 8 && mtiles * 2 * 2 * splits < 120) splits *= 2;
        const long long split_stride = 2LL * nb * 256;
        int rc = rlca_tc_gemm(pr, 2, nb, 256, FEAT, 256, splits, split_stride, s);
        if (rc) return rc;
        rlca_tc_splitk_bias_relu(pol->P, splits, split_stride, (long long)nb * 256, ta.fc1b, tc.fc1b, nb, 256, pol->X,
                                 pol->X + (size_t)nb * XLD, XLD, s);
        pol->launches += (pol->weights_dirty && !pol->w1_split_valid) ? 3 : 2;
    } else {
        // fc1: X[:, :256] = relu(F W1^T + b1)
        g.M = nb; g.N = 256; g.K = FEAT; g.lda = FEAT; g.ldb = FEAT; g.ldc = XLD; g.relu = 1;
        g.pr[0] = GemmProblem{pol->F, ta.fc1w, ta.fc1b, nullptr, pol->X};
        g.pr[1] = GemmProblem{pol->F + (size_t)nb * FEAT, tc.fc1w, tc.fc1b, nullptr, pol->X + (size_t)nb * XLD};
        launch_gemm<false, true>(g, 2, s);
    }
    fill_gs_kernel<<<(nb + 127) / 128, 128, 0, s>>>(pol->X, gs, nb);
    // fc2: H2 = relu(X W2^T + b2)
    g.M = nb; g.N = 128; g.K = XLD; g.lda = XLD; g.ldb = XLD; g.ldc = 128; g.relu = 1;
    g.pr[0] = GemmProblem{pol->X, ta.fc2w, ta.fc2b, nullptr, pol->H2};
    g.pr[1] = GemmProblem{pol->X + (size_t)nb * XLD, tc.fc2w, tc.fc2b, nullptr, pol->H2 + (size_t)nb * 128};
    launch_gemm<false, true>(g, 2, s);
    heads_fwd_kernel<<<(nb * 32 + 255) / 256, 256, 0, s>>>(
        pol->H2, params + tensor_offset(T_A1W), params + tensor_offset(T_A1B), params + tensor_offset(T_A2W),
        params + tensor_offset(T_A2B), params + tensor_offset(T_CRITW), params + tensor_offset(T_CRITB), nb, value, mean);
    pol->launches += 4;
    pol->weights_dirty = 0;
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_policy_sample(const float *params, const float *mean, int32_t nb, uint64_t seed, uint64_t counter,
                                  int32_t deterministic, float *action, float *logprob, float *scaled, void *stream)
{
    if (!params || !mean || !action || !logprob || nb < 1) return rlca_set_err(RLCA_ERR_INVALID, "NULL argument");
    sample_kernel<<<(nb + 127) / 128, 128, 0, (cudaStream_t)stream>>>(params + tensor_offset(T_LOGSTD), mean, nb, seed,
                                                                      counter, deterministic, action, logprob, scaled);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_ppo_loss_fwd_bwd(rlca_policy *pol, const float *params, const float *value, const float *mean,
                                     const float *action, const float *old_logprob, const float *adv,
                                     const float *target, int32_t nb, float clip_value, float coeff_entropy,
                                     float value_coef, float *losses, void *stream)
{
    return rlca_ppo_loss_fwd_bwd_weighted(pol, params, value, mean, action, old_logprob, adv, target, nb, clip_value,
                                          coeff_entropy, value_coef, 1.0f, losses, stream);
}

extern "C" int rlca_ppo_loss_fwd_bwd_weighted(rlca_policy *pol, const float *params, const float *value, const float *mean,
                                              const float *action, const float *old_logprob, const float *adv,
                                              const float *target, int32_t nb, float clip_value, float coeff_entropy,
                                              float value_coef, float grad_weight, float *losses, void *stream)
{
    if (!pol || !params || !value || !mean || !action || !old_logprob || !adv || !target || !losses)
        return rlca_set_err(RLCA_ERR_INVALID, "NULL argument");
    if (nb < 1 || nb > pol->max_batch) return rlca_set_err(RLCA_ERR_INVALID, "nb exceeds the workspace max_batch");
    ppo_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(params + tensor_offset(T_LOGSTD), value, mean, action,
                                                         old_logprob, adv, target, nb, clip_value, coeff_entropy,
                                                         value_coef, grad_weight, pol->dOut, losses, pol->red);
    pol->launches += 1;
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_bc_loss_fwd_bwd(rlca_policy *pol, const float *params, const float *mean,
                                    const float *target_action, int32_t nb, float *losses, void *stream)
{
    if (!pol || !params || !mean || !target_action || !losses) return rlca_set_err(RLCA_ERR_INVALID, "NULL argument");
    if (nb < 1 || nb > pol->max_batch) return rlca_set_err(RLCA_ERR_INVALID, "nb exceeds the workspace max_batch");
    bc_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(mean, target_action, nb, pol->dOut, losses, pol->red);
    pol->launches += 1;
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_policy_backward(rlca_policy *pol, const float *params, const float *obs, const float *gs, int32_t nb,
                                    float *grads, void *stream)
{
    (void)gs;
    if (!pol || !params || !obs || !grads) return rlca_set_err(RLCA_ERR_INVALID, "NULL argument");
    if (nb < 1 || nb > pol->max_batch) return rlca_set_err(RLCA_ERR_INVALID, "nb exceeds the workspace max_batch");
    cudaStream_t s = (cudaStream_t)stream;
    const TowerPtrs ta = tower_ptrs(params, 0), tc = tower_ptrs(params, 1);
    const TowerGrads ga = tower_grads(grads, 0), gc = tower_grads(grads, 1);
    const size_t B = (size_t)nb;
    // padding floats between tensors must stay zero for the optimizer / all-reduce
    RLCA_CUDA_TRY(cudaMemsetAsync(grads, 0, sizeof(float) * (size_t)tensor_offset(RLCA_POLICY_NTENSORS), s));
    RLCA_CUDA_TRY(cudaMemcpyAsync(grads + tensor_offset(T_LOGSTD), pol->red, 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    // Streams: s carries the chain the conv towers wait for (heads -> dX -> split of dZ1 -> dF); s0 the transposed split
    // of F (needs only the forward) and the dW_fc1 GEMM; s1 the small weight / bias gradients.  One stream when the
    // tensor-core path is off, on request, or while a data-parallel caller waits on fc_grads_event.
    const bool side = pol->use_side && pol->use_tc && !pol->fc_grads_event;
    cudaStream_t s0 = side ? pol->side[0] : s, s1 = side ? pol->side[1] : s;
    const size_t WSZ = (size_t)256 * FEAT;
    const size_t BP = (size_t)((nb + 31) / 32 * 32);
    RlcaTcProblem pw[2], pf[2];
    const float *dzsrc[2], *fsrc[2];
    float *dzh[2], *dzl[2], *dzth[2], *dztl[2], *fth[2], *ftl[2];
    for (int t = 0; t < 2; ++t) {
        dzsrc[t] = pol->dX + (size_t)t * B * XLD;                              // dZ1 [nb,256], pitch 260
        fsrc[t] = pol->F + (size_t)t * B * FEAT;
        dzh[t] = pol->dZs + (size_t)(2 * t) * B * 256; dzl[t] = dzh[t] + B * 256;
        dzth[t] = pol->dZTs + (size_t)(2 * t) * 256 * BP; dztl[t] = dzth[t] + 256 * BP;
        fth[t] = pol->FTs + (size_t)(2 * t) * FEAT * BP; ftl[t] = fth[t] + FEAT * BP;
        // dW_fc1 (256 x 4096) = dZ1^T F : A = dZ1^T [256, nb], B = F^T [4096, nb]
        pw[t] = RlcaTcProblem{dzth[t], dztl[t], fth[t], ftl[t], (int)BP, (int)BP, t == 0 ? ga.fc1w : gc.fc1w, nullptr};
        // dF (nb x 4096) = dZ1 W_fc1 : A = dZ1 [nb,256], B = W1^T [4096,256]; the relu(conv2) mask is applied by the
        // consumer (conv_tower_bwd) so this output-bound GEMM's epilogue is a pure coalesced store
        pf[t] = RlcaTcProblem{dzh[t], dzl[t], pol->W1Ts + (size_t)(2 * t) * WSZ, pol->W1Ts + (size_t)(2 * t + 1) * WSZ, 256, 256,
                              pol->dF + (size_t)t * B * FEAT, nullptr};
    }
    if (side) {
        RLCA_CUDA_TRY(cudaEventRecord(pol->ev_fork, s));         // after the memset of the gradient buffer
        RLCA_CUDA_TRY(cudaStreamWaitEvent(s0, pol->ev_fork, 0));
        RLCA_CUDA_TRY(cudaStreamWaitEvent(s1, pol->ev_fork, 0));
    }
    const bool tc_conv = pol->use_tc && pol->use_tc_conv && ((uintptr_t)obs & 15) == 0;
    if (tc_conv && pol->conv_bwd_dirty) {      // weight image of the conv tower backward: needs only the weights (side 1)
        const float *w1[2] = {ta.cv1w, tc.cv1w}, *b1[2] = {ta.cv1b, tc.cv1b};
        const float *w2[2] = {ta.cv2w, tc.cv2w}, *b2[2] = {ta.cv2b, tc.cv2b};
        rlca_conv_tc_bwd_prep(w1, b1, w2, b2, pol->WimgB, s1);
        if (side) RLCA_CUDA_TRY(cudaEventRecord(pol->ev_prep, s1));
        pol->launches += 1;
    }
    if (pol->use_tc && side)
        for (int t = 0; t < 2; ++t)      // one launch per tower (rather than one fused two-tower launch)
            rlca_tc_transpose_split(fsrc[t], nb, FEAT, FEAT, fth[t], ftl[t], (int)BP, s0);
    const int chunks = (nb + HEAD_CHUNK - 1) / HEAD_CHUNK;
    heads_bwd_kernel<<<chunks, 128, 0, s>>>(pol->H2, pol->dOut, params + tensor_offset(T_A1W),
                                            params + tensor_offset(T_A2W), params + tensor_offset(T_CRITW), nb, pol->dZ2,
                                            pol->headpart);
    if (side) {
        RLCA_CUDA_TRY(cudaEventRecord(pol->ev_heads, s));
        RLCA_CUDA_TRY(cudaStreamWaitEvent(s1, pol->ev_heads, 0));
    }
    heads_part_reduce_kernel<<<3, HPR_GROUPS * 132, 0, s1>>>(pol->headpart, chunks, grads + tensor_offset(T_A1W),
                                               grads + tensor_offset(T_A1B), grads + tensor_offset(T_A2W),
                                               grads + tensor_offset(T_A2B), grads + tensor_offset(T_CRITW),
                                               grads + tensor_offset(T_CRITB));
    // fc2 bias grads
    ColsumArgs cs{};
    cs.A[0] = pol->dZ2; cs.A[1] = pol->dZ2 + B * 128; cs.P = pol->S;
    cs.rows = nb; cs.cols = 128; cs.ld = 128;
    colsum_kernel<<<dim3(4, 2, RSPLIT), 256, 0, s1>>>(cs);
    reduce_splits_kernel<<<dim3(1, 2), 256, 0, s1>>>(pol->S, RSPLIT, 128, ga.fc2b, gc.fc2b);
    GemmArgs g{};
    // dW_fc2 (128 x 260) = dZ2^T X
    g.M = 128; g.N = XLD; g.K = nb; g.lda = 128; g.ldb = XLD; g.ldc = XLD; g.relu = 0;
    g.ksplit = RSPLIT; g.split_stride = 2LL * 128 * XLD;       // partial P[(split*2 + tower)][128][260]
    g.pr[0] = GemmProblem{pol->dZ2, pol->X, nullptr, nullptr, pol->S};
    g.pr[1] = GemmProblem{pol->dZ2 + B * 128, pol->X + B * XLD, nullptr, nullptr, pol->S + 128 * XLD};
    launch_gemm<true, false>(g, 2, s1);
    reduce_splits_kernel<<<dim3((128 * XLD + 255) / 256, 2), 256, 0, s1>>>(pol->S, RSPLIT, 128 * XLD, ga.fc2w, gc.fc2w);
    g.ksplit = 0; g.split_stride = 0;
    // dX (nb x 260) = dZ2 W_fc2, masked by relu(fc1) (columns 256..259 = goal/speed carry no parameter gradient)
    g.M = nb; g.N = 256; g.K = 128; g.lda = 128; g.ldb = XLD; g.ldc = XLD; g.relu = 0;
    g.pr[0] = GemmProblem{pol->dZ2, ta.fc2w, nullptr, pol->X, pol->dX};
    g.pr[1] = GemmProblem{pol->dZ2 + B * 128, tc.fc2w, nullptr, pol->X + B * XLD, pol->dX + B * XLD};
    launch_gemm<false, false>(g, 2, s);
    if (side) {
        RLCA_CUDA_TRY(cudaEventRecord(pol->ev_dx, s));
        RLCA_CUDA_TRY(cudaStreamWaitEvent(s1, pol->ev_dx, 0));
    }
    // fc1 bias grads
    cs.A[0] = pol->dX; cs.A[1] = pol->dX + B * XLD; cs.P = pol->S;
    cs.rows = nb; cs.cols = 256; cs.ld = XLD;
    colsum_kernel<<<dim3(8, 2, RSPLIT), 256, 0, s1>>>(cs);
    reduce_splits_kernel<<<dim3(1, 2), 256, 0, s1>>>(pol->S, RSPLIT, 256, ga.fc1b, gc.fc1b);
    if (side) RLCA_CUDA_TRY(cudaEventRecord(pol->ev_join[1], s1));
    if (pol->use_tc) {
        // both fc1 gradient GEMMs on the tensor cores (operands made K-major by transpose+split kernels)
        rlca_tc_split_both(dzsrc, nb, 256, XLD, dzh, dzl, 256, dzth, dztl, (int)BP, s);
        if (side) {
            RLCA_CUDA_TRY(cudaEventRecord(pol->ev_split, s));
            RLCA_CUDA_TRY(cudaStreamWaitEvent(s0, pol->ev_split, 0));
        } else {
            for (int t = 0; t < 2; ++t)
                rlca_tc_transpose_split(fsrc[t], nb, FEAT, FEAT, fth[t], ftl[t], (int)BP, s);
        }
        int rc = rlca_tc_gemm(pw, 2, 256, FEAT, nb, FEAT, 1, 0, s0);
        if (rc) return rc;
        if (side) RLCA_CUDA_TRY(cudaEventRecord(pol->ev_join[0], s0));
        // every gradient outside the conv towers (97 % of the buffer) is final here: a data-parallel caller starts their
        // all-reduce now, under the dF GEMM and the conv tower backward that follow
        if (pol->fc_grads_event) RLCA_CUDA_TRY(cudaEventRecord(pol->fc_grads_event, s));
        rc = rlca_tc_gemm(pf, 2, nb, FEAT, 256, FEAT, 1, 0, s);
        if (rc) return rc;
        pol->launches += 5;
    } else {
    // dW_fc1 (256 x 4096) = dZ1^T F
    g.M = 256; g.N = FEAT; g.K = nb; g.lda = XLD; g.ldb = FEAT; g.ldc = FEAT; g.relu = 0;
    g.pr[0] = GemmProblem{pol->dX, pol->F, nullptr, nullptr, ga.fc1w};
    g.pr[1] = GemmProblem{pol->dX + B * XLD, pol->F + B * FEAT, nullptr, nullptr, gc.fc1w};
    launch_gemm<true, false>(g, 2, s);
    if (pol->fc_grads_event) RLCA_CUDA_TRY(cudaEventRecord(pol->fc_grads_event, s));
    // dF (nb x 4096) = dZ1 W_fc1, masked by relu(conv2)
    g.M = nb; g.N = FEAT; g.K = 256; g.lda = XLD; g.ldb = FEAT; g.ldc = FEAT; g.relu = 0;
    g.pr[0] = GemmProblem{pol->dX, ta.fc1w, nullptr, pol->F, pol->dF};
    g.pr[1] = GemmProblem{pol->dX + B * XLD, tc.fc1w, nullptr, pol->F + B * FEAT, pol->dF + B * FEAT};
    launch_gemm<false, false>(g, 2, s);
    }
    if (tc_conv) {
        // conv tower backward on the tensor cores: one partial per CTA instead of one per sample
        if (pol->conv_bwd_dirty) {
            if (side) RLCA_CUDA_TRY(cudaStreamWaitEvent(s, pol->ev_prep, 0));
            pol->conv_bwd_dirty = 0;
        }
        const int bwd_sms = pol->num_sms - pol->reserved_sms > 8 ? pol->num_sms - pol->reserved_sms : pol->num_sms;
        int rc = rlca_conv_tc_backward(obs, pol->WimgB, pol->dF, pol->F, pol->part, nb, bwd_sms, s);
        if (rc) return rc;
        conv_part_reduce_kernel<<<dim3((CONV_PART + 255) / 256, 2, RSPLIT), 256, 0, s>>>(
            pol->part, rlca_conv_tc_bwd_slots(nb, bwd_sms), pol->S2);
    } else {
        if (pol->wc_dirty) {      // (a forward on the tensor-core path followed by a backward that cannot use it)
            conv_prep_weights_kernel<<<dim3((CONV_WBLK + 255) / 256, 2), 256, 0, s>>>(ta, tc, pol->Wc);
            pol->wc_dirty = 0;
            pol->launches += 1;
        }
        conv_tower_bwd_kernel<<<dim3((nb + CONV_SPC - 1) / CONV_SPC, 2), 256, sizeof(ConvBwdSmem), s>>>(
            obs, pol->Wc, ta, tc, pol->dF, pol->use_tc ? pol->F : nullptr, pol->part, nb);
        conv_part_reduce_kernel<<<dim3((CONV_PART + 255) / 256, 2, RSPLIT), 256, 0, s>>>(pol->part, nb, pol->S2);
    }
    conv_part_final_kernel<<<dim3((CONV_PART + 255) / 256, 2), 256, 0, s>>>(pol->S2, RSPLIT, ga, gc);
    if (side) {                          // the caller's stream continues (all-reduce, optimizer) when every gradient is final
        RLCA_CUDA_TRY(cudaStreamWaitEvent(s, pol->ev_join[0], 0));
        RLCA_CUDA_TRY(cudaStreamWaitEvent(s, pol->ev_join[1], 0));
    }
    pol->launches += 10;
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_adam_step(float *params, const float *grads, float *exp_avg, float *exp_avg_sq, int64_t n, float lr,
                              float beta1, float beta2, float eps, int32_t step, float grad_scale, void *stream)
{
    if (!params || !grads || !exp_avg || !exp_avg_sq || n < 1 || step < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "bad Adam arguments");
    const float bc1 = 1.0f - powf(beta1, (float)step);
    const float bc2 = 1.0f - powf(beta2, (float)step);
    adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(params, grads, exp_avg, exp_avg_sq, n, lr,
                                                                            beta1, beta2, eps, bc1, sqrtf(bc2), grad_scale);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_policy_adam_step(rlca_policy *pol, float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                                     float lr, float beta1, float beta2, float eps, int32_t step, float grad_scale,
                                     void *stream)
{
    if (!pol || !params || !grads || !exp_avg || !exp_avg_sq || step < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "bad Adam arguments");
    const int64_t n = tensor_offset(RLCA_POLICY_NTENSORS);
    const float bc1 = 1.0f - powf(beta1, (float)step);
    const float bc2 = 1.0f - powf(beta2, (float)step);
    if (pol->use_tc) {
        const size_t WSZ = (size_t)256 * FEAT;
        AdamSplitArgs a{};
        a.p = params; a.g = grads; a.m = exp_avg; a.v = exp_avg_sq; a.n = n;
        a.w_off0 = tensor_offset(T_CV1W + 4); a.w_off1 = tensor_offset(T_CRT0 + 4);
        a.hi0 = pol->W1s; a.lo0 = a.hi0 + WSZ; a.hi1 = pol->W1s + 2 * WSZ; a.lo1 = a.hi1 + WSZ;
        a.thi0 = pol->W1Ts; a.tlo0 = a.thi0 + WSZ; a.thi1 = pol->W1Ts + 2 * WSZ; a.tlo1 = a.thi1 + WSZ;
        a.lr = lr; a.b1 = beta1; a.b2 = beta2; a.eps = eps; a.bc1 = bc1; a.bc2_sqrt = sqrtf(bc2); a.grad_scale = grad_scale;
        a.tile_blocks = 2 * 8 * 128;
        const int64_t rest = n - 2 * (int64_t)WSZ;
        adam_split_kernel<<<(unsigned)(a.tile_blocks + (rest + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
    } else {
        adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(params, grads, exp_avg, exp_avg_sq, n, lr,
                                                                                beta1, beta2, eps, bc1, sqrtf(bc2), grad_scale);
    }
    RLCA_CUDA_TRY(cudaGetLastError());
    pol->weights_dirty = 1;                       // the conv weight images are still rebuilt at the next forward / backward
    pol->wimg_dirty = 1;
    pol->conv_bwd_dirty = 1;
    pol->wc_dirty = 1;
    pol->w1_split_valid = pol->use_tc ? 1 : 0;
    pol->launches += 1;
    return RLCA_OK;
}

extern "C" int rlca_gae(const float *rewards, const float *values, const float *last_value, const uint8_t *dones,
                        int32_t T, int32_t N, float gamma, float lam, float *targets, float *advs, void *stream)
{
    if (!rewards || !values || !last_value || !dones || !targets || !advs || T < 1 || N < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "bad GAE arguments");
    gae_kernel<<<(N + 31) / 32, 256, 0, (cudaStream_t)stream>>>(rewards, values, last_value, dones, T, N, (double)gamma,
                                                               (double)lam, targets, advs);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_obs_stack_push(const float *stack_in, const float *obs, const uint8_t *flags, int32_t n,
                                   int32_t beams, float *stack_out, void *stream)
{
    if (!stack_in || !obs || !stack_out || n < 1 || beams < 4 || (beams & 3))
        return rlca_set_err(RLCA_ERR_INVALID, "bad obs_stack_push arguments");
    const int b4 = beams / 4;
    const int64_t total = (int64_t)n * b4;
    obs_stack_push_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4 *>(stack_in), reinterpret_cast<const float4 *>(obs), flags, n, b4,
        reinterpret_cast<float4 *>(stack_out));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}
