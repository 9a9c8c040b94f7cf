// rlca_gemm_tc.cu — fp32-accurate tensor-core GEMM for the fc1 layer (sm_90a: wgmma + TMA + mbarriers).
//
//   C[M,N] = A[M,K] . B[N,K]^T          (both operands K-major, fp32 in HBM)
//
// fc1 (4096 -> 256) holds 66 % of the policy's FLOPs and 97 % of its parameters (SURVEY.md §2b).  The
// north-star budget (losses within 1e-4 of the fp32 reference) rules out plain TF32/BF16 over K = 4096, so
// the kernel runs "3xTF32": every operand is split on the fly into hi = tf32(x) and lo = x - hi (both exactly
// representable), and D += A_hi B_hi + A_lo B_hi + A_hi B_lo on the tensor cores with fp32 accumulation in
// registers; the dropped lo*lo term is ~2^-22 relative.
//
// Structure (one CTA per 128 x BLOCK_N output tile and K split; 3 warpgroups):
//   warpgroup 0     TMA producer (one thread): 4 tiles per k-block (A_hi, A_lo, B_hi, B_lo; 128B-swizzled,
//                   32 fp32 per row) through a 3-stage full/empty mbarrier ring
//   warpgroups 1-2  consumers, rows 0..63 / 64..127 of the tile: 12 wgmma.m64n128k8 tf32 per k-block, one
//                   commit group in flight; a stage is released once the group that read it has retired.
//                   Epilogue: registers -> the warp's 16-row slab of the idle pipeline smem -> (optional mask)
//                   -> row-wise coalesced global stores
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"
#include "rlca_gemm_tc.cuh"
#include "rlca_tc_ptx.cuh"

using namespace rlca_ptx;

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 32;            // 32 fp32 = 128 bytes = one swizzle-128B row
constexpr int MMA_K = 8;               // tf32: 32 bytes per MMA
constexpr int STAGES = 3;
constexpr int TILE_BYTES = BLOCK_M * BLOCK_K * 4;           // 16 KB (A and B tiles have the same shape)
constexpr int STAGE_BYTES = 4 * TILE_BYTES;                 // A_hi, A_lo, B_hi, B_lo
constexpr int NUM_THREADS = 384;
constexpr int EP = BLOCK_N + 8;        // epilogue slab pitch: the fragment's float2 stores are conflict free
constexpr size_t SMEM_BYTES = (size_t)STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(8 * 16 * EP * 4 <= STAGES * STAGE_BYTES, "epilogue slabs exceed the pipeline smem");
static_assert(SMEM_BYTES <= 227 * 1024, "tc gemm exceeds the 227 KB shared-memory limit");

struct TcArgs {
    float *C[2];               // per problem (tower)
    const float *mask[2];      // optional: C = mask > 0 ? C : 0 (same ld as C); only with one K split
    int M, N, K, ldc;
    int k_splits;
    long long split_stride;    // elements between consecutive K-split partial outputs
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
tf32x3_gemm_kernel(const __grid_constant__ CUtensorMap mAh0, const __grid_constant__ CUtensorMap mAl0,
                   const __grid_constant__ CUtensorMap mBh0, const __grid_constant__ CUtensorMap mBl0,
                   const __grid_constant__ CUtensorMap mAh1, const __grid_constant__ CUtensorMap mAl1,
                   const __grid_constant__ CUtensorMap mBh1, const __grid_constant__ CUtensorMap mBl1, const TcArgs args)
{
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B swizzle atoms
    uint8_t *smem = reinterpret_cast<uint8_t *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + (size_t)STAGES * STAGE_BYTES);
    uint64_t *empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int prob = blockIdx.z / args.k_splits;
    const int split = blockIdx.z - prob * args.k_splits;
    const int m0 = blockIdx.y * BLOCK_M, n0 = blockIdx.x * BLOCK_N;
    const int kblocks_total = (args.K + BLOCK_K - 1) / BLOCK_K;
    const int kb_per = (kblocks_total + args.k_splits - 1) / args.k_splits;
    const int kb0 = split * kb_per;
    const int kb1 = min(kblocks_total, kb0 + kb_per);
    const int nkb = max(0, kb1 - kb0);
    const CUtensorMap *mAh = prob ? &mAh1 : &mAh0, *mAl = prob ? &mAl1 : &mAl0;
    const CUtensorMap *mBh = prob ? &mBh1 : &mBh0, *mBl = prob ? &mBl1 : &mBl0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer =====
        if (threadIdx.x == 0) {
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                const uint32_t ph = (uint32_t)(i / STAGES) & 1u;
                mbar_wait(&empty_bar[s], ph ^ 1u);
                uint8_t *st = smem + (size_t)s * STAGE_BYTES;
                mbar_expect_tx(&full_bar[s], STAGE_BYTES);
                const int k = (kb0 + i) * BLOCK_K;
                tma_load_2d(st + 0 * TILE_BYTES, mAh, &full_bar[s], k, m0);
                tma_load_2d(st + 1 * TILE_BYTES, mAl, &full_bar[s], k, m0);
                tma_load_2d(st + 2 * TILE_BYTES, mBh, &full_bar[s], k, n0);
                tma_load_2d(st + 3 * TILE_BYTES, mBl, &full_bar[s], k, n0);
            }
        }
        return;
    }
    // ===== consumers: warpgroup c = rows 64c .. 64c+63 of the tile =====
    const int c = (warp >> 2) - 1, w = warp & 3;
    float acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.0f;
    for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (uint32_t)(i / STAGES) & 1u;
        mbar_wait(&full_bar[s], ph);
        const uint32_t sbase = smem_addr(smem + (size_t)s * STAGE_BYTES);
        const uint32_t a_base = sbase + (uint32_t)c * 64 * 128;      // 64 rows of 128 bytes
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
            const uint32_t koff = (uint32_t)k * MMA_K * 4;           // bytes inside the 128B swizzle row
            const uint64_t ah = wgmma_desc_sw128(a_base + 0 * TILE_BYTES + koff);
            const uint64_t al = wgmma_desc_sw128(a_base + 1 * TILE_BYTES + koff);
            const uint64_t bh = wgmma_desc_sw128(sbase + 2 * TILE_BYTES + koff);
            const uint64_t bl = wgmma_desc_sw128(sbase + 3 * TILE_BYTES + koff);
            wgmma_tf32_n128(acc, al, bh);                            // small terms first
            wgmma_tf32_n128(acc, ah, bl);
            wgmma_tf32_n128(acc, ah, bh);
        }
        wgmma_commit();
        wgmma_wait<1>();                                             // the previous k-block's group has retired
        if (i > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(i - 1) % STAGES]);
    }
    wgmma_wait<0>();
    fence_regs(acc);
    // both consumer warpgroups are done with the pipeline smem before it becomes the epilogue slabs
    named_bar_sync(1, 256);
    // registers -> this warp's 16 x 128 slab (pitch EP) -> row-wise, fully coalesced 512-byte global stores (and mask
    // loads): storing the fragment directly would touch 8 rows per instruction
    float *slab = reinterpret_cast<float *>(smem) + (size_t)(c * 4 + w) * 16 * EP;
#pragma unroll
    for (int j = 0; j < 64; j += 2)
        *reinterpret_cast<float2 *>(slab + (frag_row(0, lane, j)) * EP + frag_col(lane, j)) = make_float2(acc[j], acc[j + 1]);
    __syncwarp();
    float *Cp = (prob ? args.C[1] : args.C[0]) + (size_t)split * args.split_stride;
    const float *Mp = prob ? args.mask[1] : args.mask[0];
    const int n = n0 + lane * 4;
#pragma unroll 4
    for (int i = 0; i < 16; ++i) {
        const int m = m0 + c * 64 + w * 16 + i;
        if (m >= args.M) break;
        float4 v = *reinterpret_cast<const float4 *>(slab + i * EP + lane * 4);
        float *dst = Cp + (size_t)m * args.ldc + n;
        if (n + 4 <= args.N) {
            if (Mp) {
                const float4 mk = *reinterpret_cast<const float4 *>(Mp + (size_t)m * args.ldc + n);
                v.x = mk.x > 0.f ? v.x : 0.f; v.y = mk.y > 0.f ? v.y : 0.f;
                v.z = mk.z > 0.f ? v.z : 0.f; v.w = mk.w > 0.f ? v.w : 0.f;
            }
            *reinterpret_cast<float4 *>(dst) = v;
        } else {
            const float vv[4] = {v.x, v.y, v.z, v.w};
            for (int j = 0; j < 4 && n + j < args.N; ++j)
                dst[j] = (Mp && !(Mp[(size_t)m * args.ldc + n + j] > 0.f)) ? 0.f : vv[j];
        }
    }
}

// ---------------------------------------------------------------------------------------------- helpers
// split(x): hi = x with the low 13 mantissa bits cleared (exact tf32), lo = x - hi (exact).
// dst_{hi,lo}[c][r] = split(src[r][c]); 32x32 tiles through shared memory; dst rows padded to ld_out (zeros beyond rows)
__global__ void transpose_split_kernel(const float *__restrict__ src, int rows, int cols, int ld, float *__restrict__ hi,
                                       float *__restrict__ lo, int ld_out)
{
    __shared__ float tile[32][33];
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < rows && c < cols) ? src[(size_t)r * ld + c] : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;       // output row = source column
        if (c < cols && r < ld_out) {
            const float x = tile[threadIdx.x][i];
            const float h = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
            hi[(size_t)c * ld_out + r] = h;
            lo[(size_t)c * ld_out + r] = x - h;
        }
    }
}

// One pass over a [rows, cols] matrix (both towers: blockIdx.z) that writes its tf32 hi/lo split in the source layout
// AND transposed ([cols, rows], pitch ldt): the fc1 weight feeds the forward GEMM as [256, 4096] and the dF GEMM
// as [4096, 256], and both copies are rebuilt after every optimizer step.
struct SplitBothArgs {
    const float *src0, *src1;           // (selected with ?: - indexing a kernel parameter array forces a local copy)
    float *hi0, *hi1, *lo0, *lo1, *thi0, *thi1, *tlo0, *tlo1;
    int rows, cols, ld, ldo, ldt;      // source pitch, hi/lo pitch, transposed pitch (hi/lo may be NULL: transposed only)
};
__global__ void split_both_kernel(const SplitBothArgs a)
{
    __shared__ float tile[32][33];
    const int t = blockIdx.z, r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    const float *src = t ? a.src1 : a.src0;
    float *hi = t ? a.hi1 : a.hi0, *lo = t ? a.lo1 : a.lo0, *thi = t ? a.thi1 : a.thi0, *tlo = t ? a.tlo1 : a.tlo0;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        float x = 0.0f;
        if (r < a.rows && c < a.cols) {
            x = src[(size_t)r * a.ld + c];
            if (hi) {
                const float h = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
                hi[(size_t)r * a.ldo + c] = h;
                lo[(size_t)r * a.ldo + c] = x - h;
            }
        }
        tile[i][threadIdx.x] = x;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (c < a.cols && r < a.ldt) {
            const float x = tile[threadIdx.x][i];
            const float h = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
            thi[(size_t)c * a.ldt + r] = h;
            tlo[(size_t)c * a.ldt + r] = x - h;
        }
    }
}

// X[t][m][n] = relu(sum_s P[s][t][m][n] + bias[t][n])   (fc1 epilogue after a split-K GEMM)
// One thread per 4 columns of a row; rows and column groups are flattened over grid x (grid y is limited to 65535,
// and a forward may have more rows than that).  N is a multiple of 4.
__global__ void splitk_bias_relu_kernel(const float *__restrict__ P, int splits, long long split_stride,
                                        long long tower_stride, const float *__restrict__ bias0,
                                        const float *__restrict__ bias1, int M, int N, float *__restrict__ X0,
                                        float *__restrict__ X1, int ldx)
{
    const int q = N / 4, t = blockIdx.z;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)M * q) return;
    const int m = (int)(idx / q), n4 = (int)(idx - (long long)m * q) * 4;
    const float *p = P + (size_t)t * tower_stride + (size_t)m * N + n4;
    float4 acc = *reinterpret_cast<const float4 *>(p);
    for (int s = 1; s < splits; ++s) {
        const float4 v = *reinterpret_cast<const float4 *>(p + (size_t)s * split_stride);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    const float4 b = *reinterpret_cast<const float4 *>((t ? bias1 : bias0) + n4);
    float *x = (t ? X1 : X0) + (size_t)m * ldx + n4;
    *reinterpret_cast<float4 *>(x) =
        make_float4(fmaxf(acc.x + b.x, 0.f), fmaxf(acc.y + b.y, 0.f), fmaxf(acc.z + b.z, 0.f), fmaxf(acc.w + b.w, 0.f));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int get_encode()
{
    if (g_encode) return RLCA_OK;
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn)
        return rlca_set_err(RLCA_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable: %s", cudaGetErrorString(e));
    g_encode = (EncodeTiledFn)fn;
    return RLCA_OK;
}

// 2-D fp32 tensor [rows, k] with row pitch ld (floats), box = 32 x 128, 128B swizzle, zero fill out of bounds
int make_map(CUtensorMap *map, const float *base, int rows, int k, int ld)
{
    cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
    cuuint32_t box[2] = {BLOCK_K, BLOCK_M};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return rlca_set_err(RLCA_ERR_CUDA, "cuTensorMapEncodeTiled failed");
    return RLCA_OK;
}

}  // namespace

int rlca_tc_init()
{
    int rc = get_encode();
    if (rc) return rc;
    cudaError_t e = cudaFuncSetAttribute(tf32x3_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
    if (e != cudaSuccess) return rlca_set_err(RLCA_ERR_CUDA, "cudaFuncSetAttribute(tf32x3_gemm_kernel): %s", cudaGetErrorString(e));
    return RLCA_OK;
}

int rlca_tc_gemm(const RlcaTcProblem *pr, int nprob, int M, int N, int K, int ldc, int k_splits, long long split_stride,
                 cudaStream_t s)
{
    if (nprob < 1 || nprob > 2) return rlca_set_err(RLCA_ERR_INVALID, "tc gemm: nprob must be 1 or 2");
    CUtensorMap maps[8];
    memset(maps, 0, sizeof(maps));
    for (int p = 0; p < 2; ++p) {
        const RlcaTcProblem &q = pr[p < nprob ? p : 0];
        int rc = make_map(&maps[4 * p + 0], q.A_hi, M, K, q.lda); if (rc) return rc;
        rc = make_map(&maps[4 * p + 1], q.A_lo, M, K, q.lda); if (rc) return rc;
        rc = make_map(&maps[4 * p + 2], q.B_hi, N, K, q.ldb); if (rc) return rc;
        rc = make_map(&maps[4 * p + 3], q.B_lo, N, K, q.ldb); if (rc) return rc;
    }
    TcArgs a{};
    for (int p = 0; p < 2; ++p) { a.C[p] = pr[p < nprob ? p : 0].C; a.mask[p] = pr[p < nprob ? p : 0].mask; }
    a.M = M; a.N = N; a.K = K; a.ldc = ldc; a.k_splits = k_splits; a.split_stride = split_stride;
    dim3 grid((N + BLOCK_N - 1) / BLOCK_N, (M + BLOCK_M - 1) / BLOCK_M, nprob * k_splits);
    tf32x3_gemm_kernel<<<grid, NUM_THREADS, SMEM_BYTES, s>>>(maps[0], maps[1], maps[2], maps[3], maps[4], maps[5], maps[6],
                                                          maps[7], a);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

void rlca_tc_transpose_split(const float *src, int rows, int cols, int ld, float *hi, float *lo, int ld_out, cudaStream_t s)
{
    dim3 grid((cols + 31) / 32, (ld_out + 31) / 32);
    transpose_split_kernel<<<grid, dim3(32, 8), 0, s>>>(src, rows, cols, ld, hi, lo, ld_out);
}

void rlca_tc_split_both(const float *const src[2], int rows, int cols, int ld, float *const hi[2], float *const lo[2],
                        int ldo, float *const thi[2], float *const tlo[2], int ldt, cudaStream_t s)
{
    SplitBothArgs a;
    a.src0 = src[0]; a.src1 = src[1]; a.thi0 = thi[0]; a.thi1 = thi[1]; a.tlo0 = tlo[0]; a.tlo1 = tlo[1];
    a.hi0 = hi ? hi[0] : nullptr; a.hi1 = hi ? hi[1] : nullptr; a.lo0 = lo ? lo[0] : nullptr; a.lo1 = lo ? lo[1] : nullptr;
    a.rows = rows; a.cols = cols; a.ld = ld; a.ldo = ldo; a.ldt = ldt;
    dim3 grid((cols + 31) / 32, (rows + 31) / 32, 2);
    split_both_kernel<<<grid, dim3(32, 8), 0, s>>>(a);
}

void rlca_tc_splitk_bias_relu(const float *P, int splits, long long split_stride, long long tower_stride,
                              const float *bias0, const float *bias1, int M, int N, float *X0, float *X1, int ldx,
                              cudaStream_t s)
{
    const long long items = (long long)M * (N / 4);
    dim3 grid((unsigned)((items + 255) / 256), 1, 2);
    splitk_bias_relu_kernel<<<grid, 256, 0, s>>>(P, splits, split_stride, tower_stride, bias0, bias1, M, N, X0, X1, ldx);
}
