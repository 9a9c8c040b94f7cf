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

// angle wrap of the numerics contract: at most one step of 2 pi towards (-pi, pi]
__host__ __device__ __forceinline__ float dev_normalize(float a)
{
    const float pi_f = 3.14159274101257324219f;
    const float two_pi_f = 6.28318548202514648438f;
    if (a > pi_f) a -= two_pi_f;
    else if (a <= -pi_f) a += two_pi_f;
    return a;
}

// high 32 bits of a * b
__host__ __device__ __forceinline__ uint32_t dev_umulhi(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

// Philox-4x32-10 on the counter c with key (k0, k1)
__host__ __device__ __forceinline__ void dev_philox(uint32_t (&c)[4], uint32_t k0, uint32_t k1)
{
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        uint32_t hi0 = dev_umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
        uint32_t hi1 = dev_umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
        uint32_t n0 = hi1 ^ c[1] ^ k0;
        uint32_t n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}

// Four uniforms in [0, 1) (24 bits each) keyed by (seed, agent, episode, draw, purpose).  Purposes: 1 spawn and
// heading, 2 goal (rlca_env.cu); 3 start, 4 goal, 5 heading of a random layout (rlca_layout.cu).  The action sampler
// (sample_kernel, rlca_policy.cu) calls dev_philox directly with purpose word 0x5A17 and counter (row, call counter).
__host__ __device__ __forceinline__ void dev_rand4(uint64_t seed, uint32_t agent, uint32_t episode, uint32_t draw,
                                                   uint32_t purpose, float (&u)[4])
{
    uint32_t c[4] = { agent, episode, draw, purpose };
    dev_philox(c, (uint32_t)seed, (uint32_t)(seed >> 32));
#pragma unroll
    for (int i = 0; i < 4; ++i) u[i] = (float)(c[i] >> 8) * 5.9604644775390625e-08f;
}

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

// atan2(y, x) in (-pi, pi] under the same contract: the cephes atanf polynomial on min / max of |x|, |y| (reduced once
// more above tan(pi/8)), then the octant and quadrant fix-ups.  +0 and -0 for y both give pi on the negative x axis;
// atan2(0, 0) = 0.
__host__ __device__ __forceinline__ float dev_atan2f(float y, float x)
{
    const float pio2 = 1.57079632679489662f, pio4 = 0.785398163397448310f, pi = 3.14159265358979324f;
    const float ax = fabsf(x), ay = fabsf(y), hi = fmaxf(ax, ay);
    if (!(hi > 0.0f)) return 0.0f;
    float t = fminf(ax, ay) / hi, base = 0.0f;
    if (t > 0.4142135623730950f) {
        base = pio4;
        t = (t - 1.0f) / (t + 1.0f);
    }
    const float z = t * t;
    float p = fmaf(z, 8.05374449538e-2f, -1.38776856032e-1f);
    p = fmaf(p, z, 1.99777106478e-1f);
    p = fmaf(p, z, -3.33329491539e-1f);
    float a = base + fmaf(p * z, t, t);
    if (ay > ax) a = pio2 - a;
    if (x < 0.0f) a = pi - a;
    return y < 0.0f ? -a : a;
}

// natural logarithm of a positive normal x under the same contract: the cephes logf polynomial on the mantissa reduced
// to [sqrt(1/2), sqrt(2)), explicit FMAs only, so host and device round alike (about 1 ulp from the exact value).
#include <string.h>
__host__ __device__ __forceinline__ float dev_logf(float x)
{
    uint32_t b;
#ifdef __CUDA_ARCH__
    b = __float_as_uint(x);
#else
    memcpy(&b, &x, sizeof(b));
#endif
    int e = (int)(b >> 23) - 127;
    b = (b & 0x007FFFFFu) | 0x3F800000u;
    float m;
#ifdef __CUDA_ARCH__
    m = __uint_as_float(b);
#else
    memcpy(&m, &b, sizeof(m));
#endif
    if (m > 1.41421356237309505f) {
        m *= 0.5f;
        e += 1;
    }
    const float f = m - 1.0f, z = f * f, fe = (float)e;
    float p = fmaf(7.0376836292e-2f, f, -1.1514610310e-1f);
    p = fmaf(p, f, 1.1676998740e-1f);
    p = fmaf(p, f, -1.2420140846e-1f);
    p = fmaf(p, f, 1.4249322787e-1f);
    p = fmaf(p, f, -1.6668057665e-1f);
    p = fmaf(p, f, 2.0000714765e-1f);
    p = fmaf(p, f, -2.4999993993e-1f);
    p = fmaf(p, f, 3.3333331174e-1f);
    float y = fmaf(p * f, z, fe * -2.12194440e-4f);
    y = fmaf(-0.5f, z, y);
    return fmaf(fe, 0.693359375f, f + y);
}

// e^x under the same contract (crowd, DESIGN.md §9t): n = floor(x log2(e) + 1/2), r = x - n ln 2 in two parts, the
// cephes expf polynomial on r (explicit FMAs only), then 2^n applied as two exact power-of-two scalings (2^n alone
// overflows the exponent field at n = 128).  +inf above ln(FLT_MAX), 0 below ln(FLT_MIN); NaN stays NaN.
__host__ __device__ __forceinline__ float dev_expf(float x)
{
    if (x > 88.7228394f) return INFINITY;
    if (!(x >= -87.3365448f)) return x != x ? x : 0.0f;
    const float n = floorf(fmaf(x, 1.44269504088896341f, 0.5f));
    float r = fmaf(-n, 0.693359375f, x);
    r = fmaf(-n, -2.12194440e-4f, r);
    const float z = r * r;
    float p = fmaf(1.9875691500e-4f, r, 1.3981999507e-3f);
    p = fmaf(p, r, 8.3334519073e-3f);
    p = fmaf(p, r, 4.1665795894e-2f);
    p = fmaf(p, r, 1.6666665459e-1f);
    p = fmaf(p, r, 5.0000001201e-1f);
    p = fmaf(p, z, r) + 1.0f;
    const int k = (int)n, k1 = k >> 1, k2 = k - k1;
    const uint32_t b1 = (uint32_t)(k1 + 127) << 23, b2 = (uint32_t)(k2 + 127) << 23;
    float s1, s2;
#ifdef __CUDA_ARCH__
    s1 = __uint_as_float(b1);
    s2 = __uint_as_float(b2);
#else
    memcpy(&s1, &b1, sizeof(s1));
    memcpy(&s2, &b2, sizeof(s2));
#endif
    return p * s1 * s2;
}

// Box-Muller on the Philox words (a, b) (noise, DESIGN.md §9p; localization, §9s): u1 = ((a >> 8) + 1) 2^-24 in
// (0, 1], u2 = (b >> 8) 2^-24
__host__ __device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float &z0, float &z1)
{
    const float u1 = ((float)(a >> 8) + 1.0f) * 5.9604644775390625e-08f;
    const float u2 = (float)(b >> 8) * 5.9604644775390625e-08f;
    const float rho = sqrtf(-2.0f * dev_logf(u1));
    float s, c;
    dev_sincosf(6.28318548202514648438f * u2, s, c);
    z0 = rho * c;
    z1 = rho * s;
}

// the policy's goal / speed input: the goal in the robot's frame (heading sin s, cos c) and the last command (the tick,
// rlca_env.cu; the believed goal of localization, §9s)
__host__ __device__ __forceinline__ float4 goal_speed(const float4 &pose, const float4 &goal, float s, float c)
{
    const float ddx = goal.x - pose.x, ddy = goal.y - pose.y;
    return make_float4(fmaf(ddx, c, ddy * s), fmaf(ddy, c, -(ddx * s)), goal.z, goal.w);
}
