// rlca_gemm_tc.cuh — internal interface of the wgmma 3xTF32 GEMM (rlca_gemm_tc.cu).
#pragma once
#include <cuda_runtime.h>

struct RlcaTcProblem {
    const float *A_hi, *A_lo;   // [M, K] K-major, row pitch lda floats (multiple of 4)
    const float *B_hi, *B_lo;   // [N, K] K-major, row pitch ldb floats
    int lda, ldb;
    float *C;                   // [M, N] row pitch ldc (+ split * split_stride)
    const float *mask;          // optional, same pitch as C
};

int rlca_tc_init();
// C = A . B^T for 1 or 2 independent problems (the two towers) in one launch; K split into k_splits partial outputs.
int rlca_tc_gemm(const RlcaTcProblem *pr, int nprob, int M, int N, int K, int ldc, int k_splits, long long split_stride,
                 cudaStream_t s);
void rlca_tc_transpose_split(const float *src, int rows, int cols, int ld, float *hi, float *lo, int ld_out, cudaStream_t s);
// both towers in one launch: hi/lo split in the source layout (pitch ldo; hi = lo = NULL skips it) and transposed
// ([cols, rows], pitch ldt, zero-filled beyond `rows`)
void rlca_tc_split_both(const float *const src[2], int rows, int cols, int ld, float *const hi[2], float *const lo[2],
                        int ldo, float *const thi[2], float *const tlo[2], int ldt, cudaStream_t s);
void rlca_tc_splitk_bias_relu(const float *P, int splits, long long split_stride, long long tower_stride,
                              const float *bias0, const float *bias1, int M, int N, float *X0, float *X1, int ldx,
                              cudaStream_t s);
