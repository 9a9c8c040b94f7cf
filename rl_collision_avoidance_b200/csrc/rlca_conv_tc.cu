// rlca_conv_tc.cu — CNNPolicy conv tower (model/net.py:21-22,42-44 of the reference) on the Hopper tensor cores.
//
//   conv1  Conv1d(3, 32, k5, s2, p1) + ReLU : 512 -> 255        conv2  Conv1d(32, 32, k3, s2, p1) + ReLU : 255 -> 128
//
// Both convolutions are dense contractions, so they run as wgmma.mma_async tf32 with the 3xTF32 split
// (x = hi + lo, D += lo*hi + hi*lo + hi*hi; fp32 accumulation in registers) that keeps fp32 accuracy.
// One persistent CTA per SM walks over samples; warpgroup t (0 actor, 1 critic) owns tower t.  Per sample:
//
//   conv1   A1 = im2col of the scan, one 128-row tile built by both warpgroups: row j holds the 15 taps (+ a constant
//           1 that multiplies the bias row of B) of the EVEN output position 2j in K columns 0..15 and of the ODD
//           position 2j+1 in columns 16..31.  B1 = [64 = tower*32 + co][16] weights|bias.  Per tower two M128 N32 K16
//           products -> D1even, D1odd: row j = position, column = channel - exactly the position-major, even/odd
//           de-interleaved layout conv2 wants as its A operand.
//   relu    the warpgroup applies ReLU to its accumulators, splits hi/lo and stores the E (even) and O (odd) tiles
//           [128 positions x 32 channels] of its tower as 128B-swizzled K-major smem tiles.
//   conv2   out[q] = W_k1 h1[2q] + W_k2 h1[2q+1] + W_k0 h1[2q-1]:   Da|Db = O.[W_k2|W_k0] (N64) then Da += E.W_k1.
//           The k0 tap is produced one row too low (row q holds W_k0 h1[2q+1]); the epilogue adds row q-1 with warp
//           shuffles (and one smem exchange per warp boundary) instead of building a shifted copy of the operand.
//   store   relu(Da + shift(Db) + b2) -> F (flatten order c*128+q) and its tf32 hi/lo split for the fc1 GEMM.
//
// wgmma takes an M64 slice per instruction, so every M128 product is two instructions (rows 0..63, 64..127).  The
// two towers' warpgroups run their MMAs and epilogues independently; they meet only around the shared A1 tile.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"
#include "rlca_conv_tc.cuh"
#include "rlca_tc_ptx.cuh"

using namespace rlca_ptx;

namespace {

constexpr int FEAT = 4096;
constexpr int TILE_F = 128 * 32;                  // floats in one [128 x 32] operand tile (16 KB)
constexpr uint32_t MHALF = 64 * 128;              // bytes between the two M64 halves of a 128-row tile
// ---- weight image (global, prepared once per weight change; float offsets).  Every tile is already 128B-swizzled.
constexpr int W_B1 = 0;                           // [64 rows = tower*32+co][32]: cols 0..15 hi(w1|b1), 16..31 lo
constexpr int W_T0 = 64 * 32;                     // per tower: B2O_hi[64][32] B2O_lo B2E_hi[32][32] B2E_lo
constexpr int W_TOWER = 2 * 64 * 32 + 2 * 32 * 32;
constexpr int W_BIAS2 = W_T0 + 2 * W_TOWER;       // [2][32] conv2 bias
constexpr int W_FLOATS = W_BIAS2 + 64;            // 14400 floats = 57600 B
// ---- shared memory (byte offsets from a 1024-aligned base)
constexpr int OFF_W = 0;
constexpr int OFF_A1 = 57 * 1024;                 // A1 hi, lo
constexpr int OFF_A2 = OFF_A1 + 2 * TILE_F * 4;   // [tower][E_hi, E_lo, O_hi, O_lo]
constexpr int XS_PITCH = 520;                     // padded scan row: xs[c][4 + i] = x[c][i], zeros around
constexpr int OFF_XS = OFF_A2 + 8 * TILE_F * 4;
constexpr int OFF_XCHG = OFF_XS + 3 * XS_PITCH * 4;   // [tower][M half][warp][32]: last row of each warp's slice
constexpr int OFF_BAR = OFF_XCHG + 2 * 2 * 4 * 32 * 4;
constexpr int SMEM_USED = OFF_BAR + 128;
constexpr size_t SMEM_BYTES = SMEM_USED + 1024;   // + alignment slack
static_assert(W_FLOATS * 4 <= OFF_A1, "weight image overlaps A1");
static_assert(SMEM_BYTES <= 227 * 1024, "conv tc kernel exceeds the 227 KB shared-memory limit");

constexpr int NTHREADS = 256;                     // two warpgroups

enum { BAR_X = 0, BAR_W = 1 };

struct ConvTcWeights {
    const float *cv1w[2], *cv1b[2], *cv2w[2], *cv2b[2];
};

__global__ void conv_tc_prep_kernel(ConvTcWeights w, float *__restrict__ img)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W_FLOATS) return;
    float val;
    int dst;
    bool lo;
    // (tower pointers selected with ?: - indexing a kernel-parameter array with a runtime value forces a local copy)
    if (i < W_T0) {
        const int n = i >> 5, c = i & 31, t = n >> 5, co = n & 31, k = c & 15;
        lo = c >= 16;
        val = k < 15 ? (t ? w.cv1w[1] : w.cv1w[0])[co * 15 + k] : (t ? w.cv1b[1] : w.cv1b[0])[co];
        dst = W_B1 + sw128_index(n, c);
    } else if (i < W_BIAS2) {
        const int r = i - W_T0, t = r / W_TOWER, q = r - t * W_TOWER;
        if (q < 2 * 64 * 32) {            // O-pass operand: rows 0..31 tap k=2 (-> Da), rows 32..63 tap k=0 (-> Db)
            lo = q >= 64 * 32;
            const int e = q & (64 * 32 - 1), n = e >> 5, ci = e & 31, co = n & 31, tap = n < 32 ? 2 : 0;
            val = (t ? w.cv2w[1] : w.cv2w[0])[co * 96 + ci * 3 + tap];
            dst = W_T0 + t * W_TOWER + (lo ? 64 * 32 : 0) + sw128_index(n, ci);
        } else {                          // E-pass operand: tap k=1
            const int q2 = q - 2 * 64 * 32;
            lo = q2 >= 32 * 32;
            const int e = q2 & (32 * 32 - 1), co = e >> 5, ci = e & 31;
            val = (t ? w.cv2w[1] : w.cv2w[0])[co * 96 + ci * 3 + 1];
            dst = W_T0 + t * W_TOWER + 2 * 64 * 32 + (lo ? 32 * 32 : 0) + sw128_index(co, ci);
        }
    } else {
        const int r = i - W_BIAS2;
        img[i] = ((r >> 5) ? w.cv2b[1] : w.cv2b[0])[r & 31];
        return;
    }
    const float h = tf32_hi(val);
    img[dst] = lo ? val - h : h;
}

// im2col row (half H: 0 = even output position 2j, 1 = odd position 2j+1) -> 4 chunks of the A1 hi / lo tiles
template <int H>
__device__ __forceinline__ void build_a1_row(const float *__restrict__ xs, float *__restrict__ a1hi, float *__restrict__ a1lo,
                                             int j)
{
    float v[16];
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
        const float4 p = *reinterpret_cast<const float4 *>(xs + ci * XS_PITCH + 4 * j);
        const float4 q = *reinterpret_cast<const float4 *>(xs + ci * XS_PITCH + 4 * j + 4);
        const float4 r = *reinterpret_cast<const float4 *>(xs + ci * XS_PITCH + 4 * j + 8);
        const float w[12] = {p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w, r.x, r.y, r.z, r.w};
        // padded index of tap kk: (2p + kk - 1) + 4 with p = 2j + H  ->  4j + 3 + 2H + kk
#pragma unroll
        for (int kk = 0; kk < 5; ++kk) v[ci * 5 + kk] = w[3 + 2 * H + kk];
    }
    v[15] = 1.0f;                      // multiplies the bias row of B1
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int idx = j * 32 + (((H * 4 + c) ^ (j & 7)) << 2);
        float4 hi, lo;
        hi.x = tf32_hi(v[4 * c + 0]); hi.y = tf32_hi(v[4 * c + 1]); hi.z = tf32_hi(v[4 * c + 2]); hi.w = tf32_hi(v[4 * c + 3]);
        lo.x = v[4 * c + 0] - hi.x; lo.y = v[4 * c + 1] - hi.y; lo.z = v[4 * c + 2] - hi.z; lo.w = v[4 * c + 3] - hi.w;
        *reinterpret_cast<float4 *>(a1hi + idx) = hi;
        *reinterpret_cast<float4 *>(a1lo + idx) = lo;
    }
}

template <int R>
__device__ __forceinline__ void zero_regs(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; ++i) d[i] = 0.0f;
}

__global__ void __launch_bounds__(NTHREADS, 1)
conv_tower_fwd_tc_kernel(const float *__restrict__ obs, const float *__restrict__ img, float *__restrict__ F,
                         float *__restrict__ Fs, int nb)
{
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the swizzle atoms, by pointer arithmetic so the compiler keeps the shared address space
    uint8_t *sm = smem_raw + ((1024u - (smem_addr(smem_raw) & 1023u)) & 1023u);
    float *wimg = reinterpret_cast<float *>(sm + OFF_W);
    float *a1hi = reinterpret_cast<float *>(sm + OFF_A1), *a1lo = a1hi + TILE_F;
    float *a2 = reinterpret_cast<float *>(sm + OFF_A2);
    float *xs = reinterpret_cast<float *>(sm + OFF_XS);
    float *xchg = reinterpret_cast<float *>(sm + OFF_XCHG);
    uint64_t *bars = reinterpret_cast<uint64_t *>(sm + OFF_BAR);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t = warp >> 2, w = warp & 3;               // tower = warpgroup; warp inside it (rows 16w.. of an M64 slice)
    if (tid == 0) {
        mbar_init(&bars[BAR_X], 1);
        mbar_init(&bars[BAR_W], 1);
        mbar_fence_init();
    }
    if (tid < 3 * 8) {                  // zero padding of the staged scan: 4 floats before and after every channel
        const int c = tid >> 3, k = tid & 7;
        xs[c * XS_PITCH + (k < 4 ? k : 512 + k)] = 0.0f;
    }
    __syncthreads();
    const int first = blockIdx.x, stride = gridDim.x;
    // the scan of sample n, three 2 KB rows, lands in xs through the bulk-copy engine (one thread issues)
    auto load_x = [&](int n) {
        mbar_expect_tx(&bars[BAR_X], 3 * 2048);
#pragma unroll
        for (int c = 0; c < 3; ++c) tma_bulk_g2s(xs + c * XS_PITCH + 4, obs + (size_t)n * 1536 + c * 512, 2048, &bars[BAR_X]);
    };
    if (tid == 0) {
        mbar_expect_tx(&bars[BAR_W], W_FLOATS * 4);
        tma_bulk_g2s(wimg, img, W_FLOATS * 4, &bars[BAR_W]);
        if (first < nb) load_x(first);
    }

    const uint32_t sA1h = smem_addr(a1hi), sA1l = smem_addr(a1lo), sW = smem_addr(wimg);
    const uint32_t sEh = smem_addr(a2 + (size_t)(t * 4 + 0) * TILE_F), sEl = sEh + TILE_F * 4;
    const uint32_t sOh = sEh + 2 * TILE_F * 4, sOl = sEh + 3 * TILE_F * 4;
    const uint32_t bOh = sW + (W_T0 + t * W_TOWER) * 4, bOl = bOh + 64 * 32 * 4;
    const uint32_t bEh = bOh + 2 * 64 * 32 * 4, bEl = bEh + 32 * 32 * 4;
    const uint32_t b1h = sW + W_B1 * 4 + (uint32_t)t * 32 * 128, b1l = b1h + 64;     // this tower's 32 rows of B1
    const float *bias2 = wimg + W_BIAS2 + t * 32;
    float *xt = xchg + t * 256;
    const int j_a1 = w * 32 + lane;                      // A1 row this thread builds (half = t)
    int it = 0;
    for (int n = first; n < nb; n += stride, ++it) {
        const uint32_t ph = (uint32_t)it & 1u;
        // ---- im2col of sample n (shared by both towers; the previous sample's conv1 has retired in both)
        __syncthreads();
        mbar_wait(&bars[BAR_X], ph);
        if (t == 0) build_a1_row<0>(xs, a1hi, a1lo, j_a1);
        else build_a1_row<1>(xs, a1hi, a1lo, j_a1);
        fence_proxy_async();
        __syncthreads();
        if (tid == 0 && n + stride < nb) load_x(n + stride);      // every thread has consumed xs
        if (it == 0) mbar_wait(&bars[BAR_W], 0);
        // ---- conv1 of tower t: d1[h][m] = rows 64m.. of D1even (h = 0) / D1odd (h = 1), N = 32 channels
        float d1[2][2][16];
#pragma unroll
        for (int h = 0; h < 2; ++h) { zero_regs(d1[h][0]); zero_regs(d1[h][1]); }
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int kb = 0; kb < 2; ++kb) {
                    const uint32_t ao = m * MHALF + (uint32_t)h * 64 + kb * 32;
                    wgmma_tf32_n32(d1[h][m], wgmma_desc_sw128(sA1l + ao), wgmma_desc_sw128(b1h + kb * 32));
                    wgmma_tf32_n32(d1[h][m], wgmma_desc_sw128(sA1h + ao), wgmma_desc_sw128(b1l + kb * 32));
                    wgmma_tf32_n32(d1[h][m], wgmma_desc_sw128(sA1h + ao), wgmma_desc_sw128(b1h + kb * 32));
                }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < 2; ++h) { fence_regs(d1[h][0]); fence_regs(d1[h][1]); }
        // ---- conv1 result -> ReLU -> E / O operand tiles of this tower
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float *th = a2 + (size_t)(t * 4 + h * 2) * TILE_F, *tl = th + TILE_F;
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int j = 0; j < 16; j += 2) {
                    const int row = 64 * m + frag_row(w, lane, j), col = frag_col(lane, j);
                    const bool pad = (h == 1 && row == 127);      // position 255 is conv2's right zero padding
                    const float x0 = pad ? 0.f : fmaxf(d1[h][m][j], 0.f), x1 = pad ? 0.f : fmaxf(d1[h][m][j + 1], 0.f);
                    const float h0 = tf32_hi(x0), h1 = tf32_hi(x1);
                    const int idx = sw128_index(row, col);
                    *reinterpret_cast<float2 *>(th + idx) = make_float2(h0, h1);
                    *reinterpret_cast<float2 *>(tl + idx) = make_float2(x0 - h0, x1 - h1);
                }
        }
        fence_proxy_async();
        named_bar_sync(1 + t, 128);
        // ---- conv2: Da | Db = O.[W_k2 | W_k0], then Da += E.W_k1
        float da[2][16], db[2][16];
#pragma unroll
        for (int m = 0; m < 2; ++m) { zero_regs(da[m]); zero_regs(db[m]); }
        wgmma_fence();
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) {
                const uint32_t o = kb * 32, a = m * MHALF + o;
                wgmma_tf32_n64(da[m], db[m], wgmma_desc_sw128(sOl + a), wgmma_desc_sw128(bOh + o));
                wgmma_tf32_n64(da[m], db[m], wgmma_desc_sw128(sOh + a), wgmma_desc_sw128(bOl + o));
                wgmma_tf32_n64(da[m], db[m], wgmma_desc_sw128(sOh + a), wgmma_desc_sw128(bOh + o));
            }
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) {
                const uint32_t o = kb * 32, a = m * MHALF + o;
                wgmma_tf32_n32(da[m], wgmma_desc_sw128(sEl + a), wgmma_desc_sw128(bEh + o));
                wgmma_tf32_n32(da[m], wgmma_desc_sw128(sEh + a), wgmma_desc_sw128(bEl + o));
                wgmma_tf32_n32(da[m], wgmma_desc_sw128(sEh + a), wgmma_desc_sw128(bEh + o));
            }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int m = 0; m < 2; ++m) { fence_regs(da[m]); fence_regs(db[m]); }
        // ---- out[q] = relu(Da[q] + Db[q-1] + b2).  Row 16w+15 of each slice (lanes 28..31, registers j with
        // (j>>1)&1) goes through smem to the next warp; the rest of row q-1 is one shuffle away.
        if (lane >= 28) {
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int j = 2; j < 16; j += (j & 1) ? 3 : 1) xt[(m * 4 + w) * 32 + frag_col(lane, j)] = db[m][j];
        }
        named_bar_sync(1 + t, 128);
        float *out = F + ((size_t)t * nb + n) * FEAT;
        float *out_hi = Fs ? Fs + ((size_t)(2 * t) * nb + n) * FEAT : nullptr;
        float *out_lo = Fs ? Fs + ((size_t)(2 * t + 1) * nb + n) * FEAT : nullptr;
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int j0 = 0; j0 < 16; j0 = (j0 & 1) ? j0 + 3 : j0 + 1) {      // j0 = 4i + e (upper 8 rows: j0 + 2)
                const int j1 = j0 + 2, co = frag_col(lane, j0);
                const float up0 = __shfl_up_sync(0xffffffffu, db[m][j0], 4);
                const float up1 = __shfl_up_sync(0xffffffffu, db[m][j1], 4);
                const float r7 = __shfl_sync(0xffffffffu, db[m][j0], 28 + (lane & 3));      // row 16w+7
                // row 16w-1: previous warp's slice, or the last row of M half 0, or conv2's left zero padding (q = 0)
                const float prev = w > 0 ? xt[(m * 4 + w - 1) * 32 + co] : (m > 0 ? xt[3 * 32 + co] : 0.0f);
                const float p0 = lane >= 4 ? up0 : prev, p1 = lane >= 4 ? up1 : r7;
                const int q0 = 64 * m + frag_row(w, lane, j0);
                const float v0 = fmaxf(da[m][j0] + p0 + bias2[co], 0.0f);
                const float v1 = fmaxf(da[m][j1] + p1 + bias2[co], 0.0f);
                out[co * 128 + q0] = v0;
                out[co * 128 + q0 + 8] = v1;
                if (Fs) {
                    const float h0 = tf32_hi(v0), h1 = tf32_hi(v1);
                    out_hi[co * 128 + q0] = h0;
                    out_lo[co * 128 + q0] = v0 - h0;
                    out_hi[co * 128 + q0 + 8] = h1;
                    out_lo[co * 128 + q0 + 8] = v1 - h1;
                }
            }
        // the exchange rows are rewritten only after the next sample's first __syncthreads
    }
}


// =====================================================================================================================
// Backward of the conv tower on the tensor cores.  One persistent CTA per (SM, tower); per sample:
//
//   conv1   recomputed exactly as in the forward kernel (N = 32: this CTA's tower only) -> h1 (even | odd)
//   P1      dh1 "pre-scatter":  Dp[q][(tap, c1)] = sum_co g2[q][co] W2[co][c1][tap]         A = G  [128 q  x 32 co]
//   P2      dW2 += sum_q HT[(tap, c1)][q] g2T[co][q]    (K = positions)                       A = HT [96 x 128 q]
//   P3      dW1 | db1 += sum_j g1T[(half, c1)][j] im2colT[(half, k)][j]   (ones column -> bias gradient)
//
// wgmma tf32 only takes K-major operands from shared memory, so the operands whose contraction index is the position
// are written TRANSPOSED: one transposed store of a warp covers 8 positions x 4 channels of the accumulator fragment
// and lands in 32 distinct banks thanks to the 128B swizzle.  Warpgroup h recomputes conv1 half h (even / odd
// positions), runs the part of P1 that half needs (tap 1 / taps 2 | 0) and keeps one accumulator across all samples
// of the CTA: warpgroup 0 dW2 (P2), warpgroup 1 dW1 | db1 (P3).  They leave once, as one partial per CTA
// (conv_part_reduce_kernel then sums <= 66 partials per tower instead of one per sample).  g2 = dF * (F > 0) is
// formed on load; g1 = dh1 * (h1 > 0) uses mask bits kept in registers from the conv1 drain.
namespace bw {
constexpr int WB_B1 = 0;                          // [32 co][32]: cols 0..15 hi(w1|b1), 16..31 lo
constexpr int WB_W2H = 32 * 32;                   // [96 = blk*32 + c1][32 co] hi, blk 0/1/2 = tap 1/2/0
constexpr int WB_W2L = WB_W2H + 96 * 32;
constexpr int WB_TOWER = WB_W2L + 96 * 32;        // 7168 floats = 28 KB per tower
constexpr int OFF_W = 0;
constexpr int OFF_A1 = WB_TOWER * 4;              // A1 hi | lo; later the same bytes hold im2colT hi | lo
constexpr int OFF_HT = OFF_A1 + 2 * TILE_F * 4;   // HT hi | lo (4 k-atoms of 96 rows each); later g1T hi | lo
constexpr int HT_ATOM = 96 * 32, HT_LO = 4 * HT_ATOM;
constexpr int G1_ATOM = 64 * 32, G1_LO = 4 * G1_ATOM;
constexpr int IM_ATOM = 32 * 32, IM_LO = 4 * IM_ATOM;
constexpr int OFF_GT = OFF_HT + 2 * HT_LO * 4;    // g2T hi | lo (4 k-atoms of 32 rows)
constexpr int GT_ATOM = 32 * 32, GT_LO = 4 * GT_ATOM;
constexpr int OFF_G = OFF_GT + 2 * GT_LO * 4;     // G hi | lo  [128 q x 32 co]
constexpr int OFF_XCHG = OFF_G + 2 * TILE_F * 4;  // [M half][warp][32]: first row of each warp's slice (tap 0)
constexpr int OFF_BAR = OFF_XCHG + 2 * 4 * 32 * 4;
constexpr int SMEM_USED = OFF_BAR + 128;
constexpr size_t SMEM_BYTES = SMEM_USED + 1024;
static_assert(SMEM_BYTES <= 227 * 1024, "conv tc backward exceeds the 227 KB shared-memory limit");
static_assert(OFF_A1 % 1024 == 0 && OFF_HT % 1024 == 0 && OFF_GT % 1024 == 0 && OFF_G % 1024 == 0, "tile alignment");
constexpr int PART = 3616;                        // cv2w 3072 | cv2b 32 | cv1w 480 | cv1b 32  (CONV_PART of rlca_policy.cu)
constexpr int ACC1_PITCH = 33;
static_assert(PART <= 2 * GT_LO && 256 * 16 + 64 * ACC1_PITCH <= 2 * TILE_F, "partial staging exceeds G / g2T");
// P2's second M64 slice reads HT rows 64..127 of a 96-row k-atom: rows 96..127 run into the next atom and, for the
// last lo atom, into g2T.  Those accumulator rows are never stored; the reads only have to stay inside the buffers.
static_assert(OFF_HT + (HT_LO + 3 * HT_ATOM) * 4 + 128 * 128 <= OFF_GT + 2 * GT_LO * 4, "P2 slice 1 overruns g2T");
}  // namespace bw

__global__ void conv_tc_bwd_prep_kernel(ConvTcWeights w, float *__restrict__ img)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
    if (i >= bw::WB_TOWER) return;
    float val;
    int dst;
    bool lo;
    if (i < bw::WB_W2H) {
        const int co = i >> 5, c = i & 31, k = c & 15;
        lo = c >= 16;
        val = k < 15 ? (t ? w.cv1w[1] : w.cv1w[0])[co * 15 + k] : (t ? w.cv1b[1] : w.cv1b[0])[co];
        dst = bw::WB_B1 + sw128_index(co, c);
    } else {
        const int r = i - bw::WB_W2H;
        lo = r >= 96 * 32;
        const int e = lo ? r - 96 * 32 : r, n = e >> 5, co = e & 31, blk = n >> 5, c1 = n & 31;
        const int tap = blk == 0 ? 1 : (blk == 1 ? 2 : 0);
        val = (t ? w.cv2w[1] : w.cv2w[0])[co * 96 + c1 * 3 + tap];
        dst = (lo ? bw::WB_W2L : bw::WB_W2H) + sw128_index(n, co);
    }
    const float h = tf32_hi(val);
    img[(size_t)t * bw::WB_TOWER + dst] = lo ? val - h : h;
}

// the 16 im2col values (15 taps + the bias one) of output position 2j + H, straight from global memory
template <int H>
__device__ __forceinline__ void load_im2col(const float *__restrict__ x, int j, float (&v)[16])
{
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
        const float *row = x + ci * 512;
        const float4 b = __ldg(reinterpret_cast<const float4 *>(row) + j);
        if (H == 0) {
            const float a = j > 0 ? __ldg(row + 4 * j - 1) : 0.0f;          // left zero padding of Conv1d
            v[ci * 5 + 0] = a; v[ci * 5 + 1] = b.x; v[ci * 5 + 2] = b.y; v[ci * 5 + 3] = b.z; v[ci * 5 + 4] = b.w;
        } else {
            const float4 c = j < 127 ? __ldg(reinterpret_cast<const float4 *>(row) + j + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
            v[ci * 5 + 0] = b.y; v[ci * 5 + 1] = b.z; v[ci * 5 + 2] = b.w; v[ci * 5 + 3] = c.x; v[ci * 5 + 4] = c.y;
        }
    }
    v[15] = 1.0f;
}

__global__ void __launch_bounds__(NTHREADS, 1)
conv_tower_bwd_tc_kernel(const float *__restrict__ obs, const float *__restrict__ img, const float *__restrict__ dF,
                         const float *__restrict__ Fm, float *__restrict__ part, int nb, int slots)
{
    using namespace bw;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *sm = smem_raw + ((1024u - (smem_addr(smem_raw) & 1023u)) & 1023u);
    float *wimg = reinterpret_cast<float *>(sm + bw::OFF_W);
    float *a1 = reinterpret_cast<float *>(sm + bw::OFF_A1);      // hi, lo at + TILE_F  (im2colT: hi, lo at + IM_LO)
    float *ht = reinterpret_cast<float *>(sm + OFF_HT);
    float *gt = reinterpret_cast<float *>(sm + OFF_GT);
    float *gq = reinterpret_cast<float *>(sm + OFF_G);       // hi, lo at + TILE_F
    float *xchg = reinterpret_cast<float *>(sm + bw::OFF_XCHG);
    uint64_t *bars = reinterpret_cast<uint64_t *>(sm + bw::OFF_BAR);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t = blockIdx.x >= slots ? 1 : 0, slot = blockIdx.x - t * slots;
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&bars[0], WB_TOWER * 4);
        tma_bulk_g2s(wimg, img + (size_t)t * WB_TOWER, WB_TOWER * 4, &bars[0]);
    }
    const int first = slot, stride = slots;
    // element-wise roles: position j, half = warpgroup (im2col half / channel half of g2); MMA roles: warpgroup g,
    // warp w inside it (fragment rows 16w.. of each M64 slice)
    const int lq = warp & 3, half = warp >> 2, g = half, w = lq;
    const int j = lq * 32 + lane, ka = lq, jc = lane;
    const uint32_t sW = smem_addr(wimg), sA1 = smem_addr(a1), sHT = smem_addr(ht), sGT = smem_addr(gt), sG = smem_addr(gq);
    float acc_b2[16];
    zero_regs(acc_b2);
    float acc2[2][16];           // warpgroup 0: dW2, rows (blk, c1) 0..63 | 64..127 (96.. unused), columns co
    float acc1[16];              // warpgroup 1: dW1 | db1, rows (half, c1), columns (half', k)
    zero_regs(acc2[0]); zero_regs(acc2[1]); zero_regs(acc1);
    int it = 0;
    for (int n = first; n < nb; n += stride, ++it) {
        // ---- im2col values of this thread's output position (kept in registers until im2colT is written)
        float v[16];
        if (half == 0) load_im2col<0>(obs + (size_t)n * 1536, j, v);
        else load_im2col<1>(obs + (size_t)n * 1536, j, v);
        // ---- g2 = dF * (F > 0) for q = j, channels half*16 ..: G row (K-major in co) and g2T (K-major in q).
        // (G / g2T were last read by P1 / P2 of the previous sample, both retired before its g1T was written.)
        {
            const size_t base = ((size_t)t * nb + n) * FEAT + (size_t)(half * 16) * 128 + j;
            float gv[16];
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                const float f = __ldg(Fm + base + c * 128), d = __ldg(dF + base + c * 128);
                gv[c] = f > 0.0f ? d : 0.0f;
                acc_b2[c] += gv[c];
            }
#pragma unroll
            for (int c4 = 0; c4 < 4; ++c4) {
                const float4 x = make_float4(gv[4 * c4], gv[4 * c4 + 1], gv[4 * c4 + 2], gv[4 * c4 + 3]);
                const float4 hi = make_float4(tf32_hi(x.x), tf32_hi(x.y), tf32_hi(x.z), tf32_hi(x.w));
                const int idx = j * 32 + (((half * 4 + c4) ^ (j & 7)) << 2);
                *reinterpret_cast<float4 *>(gq + idx) = hi;
                *reinterpret_cast<float4 *>(gq + TILE_F + idx) = make_float4(x.x - hi.x, x.y - hi.y, x.z - hi.z, x.w - hi.w);
            }
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                const int idx = ka * GT_ATOM + sw128_index(half * 16 + c, jc);
                const float hi = tf32_hi(gv[c]);
                gt[idx] = hi;
                gt[GT_LO + idx] = gv[c] - hi;
            }
        }
        // ---- A1 (aliases the previous sample's im2colT: its P3 has retired once every thread is here)
        __syncthreads();
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int idx = j * 32 + (((half * 4 + c) ^ (j & 7)) << 2);
            const float4 hi = make_float4(tf32_hi(v[4 * c]), tf32_hi(v[4 * c + 1]), tf32_hi(v[4 * c + 2]), tf32_hi(v[4 * c + 3]));
            *reinterpret_cast<float4 *>(a1 + idx) = hi;
            *reinterpret_cast<float4 *>(a1 + TILE_F + idx) =
                make_float4(v[4 * c] - hi.x, v[4 * c + 1] - hi.y, v[4 * c + 2] - hi.z, v[4 * c + 3] - hi.w);
        }
        fence_proxy_async();
        __syncthreads();
        if (it == 0) mbar_wait(&bars[0], 0);
        // ---- conv1 half g (D1 even / odd, N = 32 channels) and P1 (warpgroup 0: tap 1 -> dp; 1: taps 2 | 0 -> dp | dq)
        float d1[2][16], dp[2][16], dq[2][16];
#pragma unroll
        for (int m = 0; m < 2; ++m) { zero_regs(d1[m]); zero_regs(dp[m]); zero_regs(dq[m]); }
        wgmma_fence();
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
                const uint32_t ao = m * MHALF + (uint32_t)g * 64 + kb * 32, bh = sW + WB_B1 * 4 + kb * 32, bl = bh + 64;
                wgmma_tf32_n32(d1[m], wgmma_desc_sw128(sA1 + TILE_F * 4 + ao), wgmma_desc_sw128(bh));
                wgmma_tf32_n32(d1[m], wgmma_desc_sw128(sA1 + ao), wgmma_desc_sw128(bl));
                wgmma_tf32_n32(d1[m], wgmma_desc_sw128(sA1 + ao), wgmma_desc_sw128(bh));
            }
        if (g == 0) {
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int kb = 0; kb < 4; ++kb) {
                    const uint32_t a = m * MHALF + kb * 32, o = kb * 32;
                    wgmma_tf32_n32(dp[m], wgmma_desc_sw128(sG + TILE_F * 4 + a), wgmma_desc_sw128(sW + WB_W2H * 4 + o));
                    wgmma_tf32_n32(dp[m], wgmma_desc_sw128(sG + a), wgmma_desc_sw128(sW + WB_W2L * 4 + o));
                    wgmma_tf32_n32(dp[m], wgmma_desc_sw128(sG + a), wgmma_desc_sw128(sW + WB_W2H * 4 + o));
                }
        } else {
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int kb = 0; kb < 4; ++kb) {
                    const uint32_t a = m * MHALF + kb * 32, o = 32 * 128 + kb * 32;    // rows 32..95 of W2r
                    wgmma_tf32_n64(dp[m], dq[m], wgmma_desc_sw128(sG + TILE_F * 4 + a), wgmma_desc_sw128(sW + WB_W2H * 4 + o));
                    wgmma_tf32_n64(dp[m], dq[m], wgmma_desc_sw128(sG + a), wgmma_desc_sw128(sW + WB_W2L * 4 + o));
                    wgmma_tf32_n64(dp[m], dq[m], wgmma_desc_sw128(sG + a), wgmma_desc_sw128(sW + WB_W2H * 4 + o));
                }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int m = 0; m < 2; ++m) { fence_regs(d1[m]); fence_regs(dp[m]); fence_regs(dq[m]); }
        // ---- h1 = relu(conv1): transposed into HT (E rows 0..31 | O rows 32..63 | O shifted by one q, rows 64..95)
        uint32_t hmask[2] = {0u, 0u};
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                const int p = 64 * m + frag_row(w, lane, r), c1 = frag_col(lane, r);
                const bool pad = (g == 1 && p == 127);              // position 255 = conv2's right zero padding
                const float x = pad ? 0.0f : fmaxf(d1[m][r], 0.0f);
                hmask[m] |= (x > 0.0f ? 1u : 0u) << r;
                const float hi = tf32_hi(x), lo = x - hi;
                const int idx = (p >> 5) * HT_ATOM + sw128_index(g * 32 + c1, p & 31);
                ht[idx] = hi;
                ht[HT_LO + idx] = lo;
                if (g == 1) {
                    // row 64 + c1 holds O[q - 1]: this value belongs to column p + 1; position 127 writes the q = 0
                    // column (left padding) instead
                    const int q = p == 127 ? 0 : p + 1;
                    const int idx2 = (q >> 5) * HT_ATOM + sw128_index(64 + c1, q & 31);
                    ht[idx2] = p == 127 ? 0.0f : hi;
                    ht[HT_LO + idx2] = p == 127 ? 0.0f : lo;
                }
            }
        fence_proxy_async();
        __syncthreads();
        // ---- P2 (warpgroup 0): ACC2[(blk, c1)][co] += HT . g2T^T  (K = q = 128: 4 k-atoms x 4 k-blocks); it runs
        // while the drain below works on other registers.  M = 96 valid rows in two M64 slices: a quarter of P2's MMA
        // work (rows 96..127, read past the atom - see the static_assert at bw::OFF_GT) is discarded.
        if (g == 0) {
            wgmma_fence();
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll 1
                for (int kt = 0; kt < 4; ++kt)
#pragma unroll
                    for (int kb = 0; kb < 4; ++kb) {
                        const uint32_t ao = (uint32_t)kt * HT_ATOM * 4 + m * MHALF + kb * 32, bo = (uint32_t)kt * GT_ATOM * 4 + kb * 32;
                        wgmma_tf32_n32(acc2[m], wgmma_desc_sw128(sHT + HT_LO * 4 + ao), wgmma_desc_sw128(sGT + bo));
                        wgmma_tf32_n32(acc2[m], wgmma_desc_sw128(sHT + ao), wgmma_desc_sw128(sGT + GT_LO * 4 + bo));
                        wgmma_tf32_n32(acc2[m], wgmma_desc_sw128(sHT + ao), wgmma_desc_sw128(sGT + bo));
                    }
            wgmma_commit();
        }
        // ---- dh1 from P1, masked by relu(conv1) -> g1 (even positions: warpgroup 0, odd: warpgroup 1)
        float g1[2][16];
        if (g == 0) {
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int r = 0; r < 16; ++r) g1[m][r] = ((hmask[m] >> r) & 1u) ? dp[m][r] : 0.0f;   // g2[j] . W_k1
        } else {
            // odd position p: g2[p] . W_k2 + g2[p+1] . W_k0.  Row p+1 of the tap-0 block is one shuffle away except
            // across a warp boundary: row 16w of each slice (lanes 0..3, registers with (r>>1)&1 == 0) goes via smem.
            if (lane < 4) {
#pragma unroll
                for (int m = 0; m < 2; ++m)
#pragma unroll
                    for (int r = 0; r < 16; r += (r & 1) ? 3 : 1) xchg[(m * 4 + w) * 32 + frag_col(lane, r)] = dq[m][r];
            }
            named_bar_sync(2, 128);
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int r0 = 0; r0 < 16; r0 = (r0 & 1) ? r0 + 3 : r0 + 1) {
                    const int r1 = r0 + 2, c1 = frag_col(lane, r0);
                    const float dn0 = __shfl_down_sync(0xffffffffu, dq[m][r0], 4);
                    const float dn1 = __shfl_down_sync(0xffffffffu, dq[m][r1], 4);
                    const float r8 = __shfl_sync(0xffffffffu, dq[m][r1], lane & 3);          // row 16w+8
                    // row 16w+16: next warp's slice, or the first row of M half 1, or nothing after position 127
                    const float next = w < 3 ? xchg[(m * 4 + w + 1) * 32 + c1] : (m == 0 ? xchg[4 * 32 + c1] : 0.0f);
                    const float n0 = lane < 28 ? dn0 : r8, n1 = lane < 28 ? dn1 : next;
                    g1[m][r0] = ((hmask[m] >> r0) & 1u) ? dp[m][r0] + n0 : 0.0f;
                    g1[m][r1] = ((hmask[m] >> r1) & 1u) ? dp[m][r1] + n1 : 0.0f;
                }
        }
        // ---- g1T and im2colT overwrite HT / A1: P2 (and conv1) must have retired
        if (g == 0) {
            wgmma_wait<0>();
            fence_regs(acc2[0]); fence_regs(acc2[1]);
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                const int p = 64 * m + frag_row(w, lane, r), c1 = frag_col(lane, r);
                const int idx = (p >> 5) * G1_ATOM + sw128_index(g * 32 + c1, p & 31);
                const float hi = tf32_hi(g1[m][r]);
                ht[idx] = hi;
                ht[G1_LO + idx] = g1[m][r] - hi;
            }
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int idx = ka * IM_ATOM + sw128_index(half * 16 + k, jc);
            const float hi = tf32_hi(v[k]);
            a1[idx] = hi;
            a1[IM_LO + idx] = v[k] - hi;
        }
        fence_proxy_async();
        __syncthreads();
        // ---- P3 (warpgroup 1): ACC1[(half, c1)][(half', k)] += g1T . im2colT^T  (K = j = 128)
        if (g == 1) {
            wgmma_fence();
#pragma unroll 1
            for (int kt = 0; kt < 4; ++kt)
#pragma unroll
                for (int kb = 0; kb < 4; ++kb) {
                    const uint32_t ao = (uint32_t)kt * G1_ATOM * 4 + kb * 32, bo = (uint32_t)kt * IM_ATOM * 4 + kb * 32;
                    wgmma_tf32_n32(acc1, wgmma_desc_sw128(sHT + G1_LO * 4 + ao), wgmma_desc_sw128(sA1 + bo));
                    wgmma_tf32_n32(acc1, wgmma_desc_sw128(sHT + ao), wgmma_desc_sw128(sA1 + IM_LO * 4 + bo));
                    wgmma_tf32_n32(acc1, wgmma_desc_sw128(sHT + ao), wgmma_desc_sw128(sA1 + bo));
                }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(acc1);
        }
    }
    // =================================================================== per-CTA partial -> global
    __syncthreads();                                           // every MMA has retired; G / g2T are dead
    float *stage = gt;                                         // PART floats
    float *red = gq;                                           // [256][16] conv2-bias partials
    float *acc1s = gq + 256 * 16;                              // [64][ACC1_PITCH] dW1 | db1 accumulator
    if (g == 0) {
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                const int row = 64 * m + frag_row(w, lane, r), co = frag_col(lane, r);
                if (row < 96) {
                    const int blk = row >> 5, c1 = row & 31, tap = blk == 0 ? 1 : (blk == 1 ? 2 : 0);
                    stage[co * 96 + c1 * 3 + tap] = acc2[m][r];
                }
            }
    } else {
#pragma unroll
        for (int r = 0; r < 16; ++r) acc1s[frag_row(w, lane, r) * ACC1_PITCH + frag_col(lane, r)] = acc1[r];
    }
#pragma unroll
    for (int c = 0; c < 16; ++c) red[tid * 16 + c] = acc_b2[c];
    __syncthreads();
    if (tid < 32) {                                            // db2[co] = sum over the 128 positions
        const int hsel = tid >> 4, c = tid & 15;
        float sacc = 0.0f;
        for (int q = 0; q < 128; ++q) sacc += red[(hsel * 128 + q) * 16 + c];
        stage[3072 + tid] = sacc;
    }
    for (int i = tid; i < 32 * 16; i += NTHREADS) {           // dW1 | db1 = even half (rows 0..31, columns 0..15)
        const int c1 = i >> 4, k = i & 15;                     //           + odd half (rows 32..63, columns 16..31)
        const float val = acc1s[c1 * ACC1_PITCH + k] + acc1s[(32 + c1) * ACC1_PITCH + 16 + k];
        if (k < 15) stage[3104 + c1 * 15 + k] = val;
        else stage[3584 + c1] = val;
    }
    __syncthreads();
    float *dst = part + ((size_t)t * slots + slot) * PART;
    for (int i = tid; i < PART; i += NTHREADS) dst[i] = stage[i];
}

}  // namespace

int rlca_conv_tc_init()
{
    cudaError_t e = cudaFuncSetAttribute(conv_tower_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
    if (e != cudaSuccess)
        return rlca_set_err(RLCA_ERR_CUDA, "cudaFuncSetAttribute(conv_tower_fwd_tc_kernel): %s", cudaGetErrorString(e));
    e = cudaFuncSetAttribute(conv_tower_bwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bw::SMEM_BYTES);
    if (e != cudaSuccess)
        return rlca_set_err(RLCA_ERR_CUDA, "cudaFuncSetAttribute(conv_tower_bwd_tc_kernel): %s", cudaGetErrorString(e));
    return RLCA_OK;
}

size_t rlca_conv_tc_image_floats() { return (size_t)W_FLOATS; }

void rlca_conv_tc_prep(const float *const cv1w[2], const float *const cv1b[2], const float *const cv2w[2],
                       const float *const cv2b[2], float *img, cudaStream_t s)
{
    ConvTcWeights w;
    for (int t = 0; t < 2; ++t) { w.cv1w[t] = cv1w[t]; w.cv1b[t] = cv1b[t]; w.cv2w[t] = cv2w[t]; w.cv2b[t] = cv2b[t]; }
    conv_tc_prep_kernel<<<(W_FLOATS + 255) / 256, 256, 0, s>>>(w, img);
}

int rlca_conv_tc_forward(const float *obs, const float *img, float *F, float *Fs, int nb, int num_sms, cudaStream_t s)
{
    const int grid = nb < num_sms ? nb : num_sms;
    conv_tower_fwd_tc_kernel<<<grid, NTHREADS, SMEM_BYTES, s>>>(obs, img, F, Fs, nb);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

size_t rlca_conv_tc_bwd_image_floats() { return 2 * (size_t)bw::WB_TOWER; }

int rlca_conv_tc_bwd_slots(int nb, int num_sms)
{
    const int per_tower = num_sms / 2 > 0 ? num_sms / 2 : 1;
    return nb < per_tower ? nb : per_tower;
}

void rlca_conv_tc_bwd_prep(const float *const cv1w[2], const float *const cv1b[2], const float *const cv2w[2],
                           const float *const cv2b[2], float *img, cudaStream_t s)
{
    ConvTcWeights w;
    for (int t = 0; t < 2; ++t) { w.cv1w[t] = cv1w[t]; w.cv1b[t] = cv1b[t]; w.cv2w[t] = cv2w[t]; w.cv2b[t] = cv2b[t]; }
    conv_tc_bwd_prep_kernel<<<dim3((bw::WB_TOWER + 255) / 256, 2), 256, 0, s>>>(w, img);
}

int rlca_conv_tc_backward(const float *obs, const float *img, const float *dF, const float *Fmask, float *part, int nb,
                          int num_sms, cudaStream_t s)
{
    const int slots = rlca_conv_tc_bwd_slots(nb, num_sms);
    conv_tower_bwd_tc_kernel<<<2 * slots, NTHREADS, bw::SMEM_BYTES, s>>>(obs, img, dF, Fmask, part, nb, slots);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}
