// rlca_common.cuh — error plumbing and contract math shared by the translation units of librlca.so.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>

#include "../../include/rlca.h"

extern thread_local char rlca_g_err[512];

inline int rlca_set_err(int code, const char *fmt, const char *a = "", const char *b = "")
{
    snprintf(rlca_g_err, sizeof(rlca_g_err), fmt, a, b);
    return code;
}

#define RLCA_CUDA_TRY(expr)                                                                      \
    do {                                                                                         \
        cudaError_t e__ = (expr);                                                                \
        if (e__ != cudaSuccess)                                                                  \
            return rlca_set_err(RLCA_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__)); \
    } while (0)

// sin / cos of the numerics contract (DESIGN.md §4): explicit FMAs only, so a host build without contraction
// (-ffp-contract=off) rounds exactly as the device does.
__host__ __device__ __forceinline__ void dev_sincosf(float x, float &s, float &c)
{
    const float two_over_pi = 0.636619772367581343f;
    const float pio2_hi = 1.57079625129699707031f;
    const float pio2_lo = 7.54978941586159635335e-08f;
    float q = rintf(x * two_over_pi);
    float r = fmaf(q, -pio2_hi, x);
    r = fmaf(q, -pio2_lo, r);
    float r2 = r * r;
    float ps = fmaf(r2, -1.9515295891e-4f, 8.3321608736e-3f);
    ps = fmaf(r2, ps, -1.6666654611e-1f);
    float sr = fmaf(r * r2, ps, r);
    float pc = fmaf(r2, 2.443315711809948e-5f, -1.388731625493765e-3f);
    pc = fmaf(r2, pc, 4.166664568298827e-2f);
    float cr = fmaf(r2 * r2, pc, fmaf(r2, -0.5f, 1.0f));
    int qi = ((int)q) & 3;
    float ss = (qi & 1) ? cr : sr;
    float cc = (qi & 1) ? sr : cr;
    if (qi == 2 || qi == 3) ss = -ss;
    if (qi == 1 || qi == 2) cc = -cc;
    s = ss;
    c = cc;
}
