// rlca_safety.cu — how closely robots pass and why they crash (sm_90a), C ABI in include/rlca.h, DESIGN.md §9m.
//
// rlca_safety_track runs after each rlca_env_step and before that tick's rlca_eval_track.  Per robot and tick it takes
//   separation  the least distance between the robot's footprint rectangle and any other robot's of its world
//               (0 when two intersect), with the robot that attains it, and
//   clearance   the nearest return in metres of the scan the tick wrote,
// folds them into the running episode (minimum separation and its partner, minimum clearance, near-miss ticks), and
// writes one record per ended episode into the slot rlca_eval_track is about to fill: the episode boundaries are the
// tracker's (closed != meta_in.y, record on flags.z != 0), read from its state and never written here.  A crash gets a
// cause from the separation d0 at the poses the tick started from: d0 above the contact bound proves that no robot
// was involved (static); otherwise the cause is the robot nearest at d0.
//
// One CTA per world.  Every function the kernel calls is __host__ __device__ and the file is built without FMA
// contraction on either side, so rlca_safety_track_host (serial loops over the same functions) equals the kernel
// bit for bit.  rlca_safety_reduce sums a world's records in float64 in agent-then-record order, one thread per world
// (and role), as rlca_eval_reduce does.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define SAFETY_THREADS 256
#define SAFETY_WARPS (SAFETY_THREADS / 32)
#define REDUCE_THREADS 128
#define MAXR RLCA_MAX_ROBOTS_PER_WORLD

// per-robot bits of one tick
#define ROBOT_TRACKED 1      // the tick belongs to an episode the tracker has not closed
#define ROBOT_RESPAWNED 2    // flags.w: state_out holds the next episode's pose
#define ROBOT_CRASHED 4      // flags.z == 2: the episode ends with result Crashed

struct SafetyParams {
    float half_len, half_wid, range_max, near_dist, contact;
    int R, beams, episodes;
};

// separation in the high word, the other robot in the low one: separations are >= 0, so their bits order as integers,
// and the low word breaks ties towards the lowest index
#define PACK_NONE 0x7f800000ffffffffull      // +inf, robot -1

__host__ __device__ __forceinline__ unsigned long long pack_sep(float s, int other)
{
    uint32_t b;
#ifdef __CUDA_ARCH__
    b = __float_as_uint(s);
#else
    memcpy(&b, &s, 4);
#endif
    return ((unsigned long long)b << 32) | (uint32_t)other;
}
__host__ __device__ __forceinline__ float packed_sep(unsigned long long p)
{
    const uint32_t b = (uint32_t)(p >> 32);
    float s;
#ifdef __CUDA_ARCH__
    s = __uint_as_float(b);
#else
    memcpy(&s, &b, 4);
#endif
    return s;
}

// the four footprint corners of pose (x, y, theta), counter-clockwise from (-half_len, -half_wid): the tick's formula
__host__ __device__ __forceinline__ void footprint(const SafetyParams &q, float4 p, float2 *c)
{
    float s, co;
    dev_sincosf(p.z, s, co);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float hx = (k == 1 || k == 2) ? q.half_len : -q.half_len;
        const float hy = (k >= 2) ? q.half_wid : -q.half_wid;
        c[k] = make_float2(fmaf(hx, co, fmaf(-hy, s, p.x)), fmaf(hx, s, fmaf(hy, co, p.y)));
    }
}

// do the projections of A and B onto edge k -> k + 1 of P leave a gap?  (a rectangle's edge directions are its
// edge normals)
__host__ __device__ __forceinline__ bool axis_separates(const float2 *P, int k, const float2 *A, const float2 *B)
{
    const float dx = P[k + 1].x - P[k].x, dy = P[k + 1].y - P[k].y;
    float a0 = INFINITY, a1 = -INFINITY, b0 = INFINITY, b1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float pa = A[i].x * dx + A[i].y * dy, pb = B[i].x * dx + B[i].y * dy;
        a0 = fminf(a0, pa);
        a1 = fmaxf(a1, pa);
        b0 = fminf(b0, pb);
        b1 = fmaxf(b1, pb);
    }
    return a1 < b0 || b1 < a0;
}

// squared distance from p to the segment a -> b
__host__ __device__ __forceinline__ float point_segment_sq(float2 p, float2 a, float2 b)
{
    const float ex = b.x - a.x, ey = b.y - a.y, wx = p.x - a.x, wy = p.y - a.y;
    float t = (wx * ex + wy * ey) / (ex * ex + ey * ey);
    t = fminf(fmaxf(t, 0.0f), 1.0f);
    const float dx = wx - t * ex, dy = wy - t * ey;
    return dx * dx + dy * dy;
}

// Distance between the rectangles A and B, 0 when no edge direction of either separates them; otherwise the least
// of the 32 corner-to-edge distances: corner i of A against edge k of B (i, then k), then B's corners against A's
// edges.  One square root, of the least squared distance.
__host__ __device__ __forceinline__ float separation(const float2 *A, const float2 *B)
{
    if (!(axis_separates(A, 0, A, B) || axis_separates(A, 1, A, B) || axis_separates(B, 0, A, B) ||
          axis_separates(B, 1, A, B)))
        return 0.0f;
    float m = INFINITY;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) m = fminf(m, point_segment_sq(A[i], B[k], B[(k + 1) & 3]));
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) m = fminf(m, point_segment_sq(B[i], A[k], A[(k + 1) & 3]));
    return sqrtf(m);
}

__host__ __device__ __forceinline__ float clearance_metres(const SafetyParams &q, float obs_min)
{
    return (obs_min + 0.5f) * q.range_max;      // the hybrid controller's nearest return (rlca_orca.cu)
}

__host__ __device__ __forceinline__ int robot_bits(uchar4 fl, int closed, int episode)
{
    return (closed != episode ? ROBOT_TRACKED : 0) | (fl.w ? ROBOT_RESPAWNED : 0) | (fl.z == 2 ? ROBOT_CRASHED : 0);
}

// Which of the pair's two separations the fold will read: at the poses the tick ended at, for a tracked robot that was
// not re-spawned; at the poses it started from, for a tracked robot that was re-spawned (its tick separation) or
// crashed (d0).
__host__ __device__ __forceinline__ bool needs_out(int ba, int bb)
{
    return ((ba & ROBOT_TRACKED) && !(ba & ROBOT_RESPAWNED)) || ((bb & ROBOT_TRACKED) && !(bb & ROBOT_RESPAWNED));
}
__host__ __device__ __forceinline__ bool needs_in(int ba, int bb)
{
    return ((ba & ROBOT_TRACKED) && (ba & (ROBOT_RESPAWNED | ROBOT_CRASHED))) ||
           ((bb & ROBOT_TRACKED) && (bb & (ROBOT_RESPAWNED | ROBOT_CRASHED)));
}

// The running episode of one robot, folded with one tick; the record goes into the tracker's next slot.
__host__ __device__ __forceinline__ void fold(const SafetyParams &q, uchar4 fl, int bits, unsigned long long tick,
                                              unsigned long long start, float clear, int32_t count, float *min_sep,
                                              float *min_clear, float *last_clear, int32_t *near, int32_t *partner,
                                              float4 *records)
{
    float ms = *min_sep, mc = *min_clear;
    int32_t nr = *near, pa = *partner;
    if (bits & ROBOT_TRACKED) {
        const float s = packed_sep(tick);
        if (s < ms) {
            ms = s;
            pa = (int32_t)(uint32_t)tick;
        }
        if (!(bits & ROBOT_RESPAWNED)) mc = fminf(mc, clear);      // a re-spawned robot's scan is the next episode's
        nr += s < q.near_dist;
        if (fl.z != 0) {
            if (count < q.episodes) {
                int cause = 0, hit = -1;
                if (bits & ROBOT_CRASHED) {
                    if (packed_sep(start) > q.contact) cause = 1;
                    else {
                        cause = 2 | (*last_clear < q.contact ? 4 : 0);
                        hit = (int32_t)(uint32_t)start;
                    }
                }
                *records = make_float4(ms, mc, (float)nr, (float)(cause | (hit + 1) << 8 | (pa + 1) << 16));
            }
            bits |= ROBOT_RESPAWNED;                                // the episode is over: start afresh
        }
    }
    if (bits & ROBOT_RESPAWNED) {
        ms = INFINITY;
        mc = INFINITY;
        nr = 0;
        pa = -1;
    }
    *min_sep = ms;
    *min_clear = mc;
    *near = nr;
    *partner = pa;
    *last_clear = clear;
}

__global__ void __launch_bounds__(SAFETY_THREADS) rlca_safety_track_kernel(
    SafetyParams q, const float4 *__restrict__ pose_in, const int4 *__restrict__ meta_in,
    const float4 *__restrict__ pose_out, const uchar4 *__restrict__ flags, const float *__restrict__ obs,
    const int32_t *__restrict__ closed, const int32_t *__restrict__ count, float *__restrict__ min_sep,
    float *__restrict__ min_clear, float *__restrict__ last_clear, int32_t *__restrict__ near,
    int32_t *__restrict__ partner, float4 *__restrict__ records)
{
    __shared__ float2 c_in[MAXR][4], c_out[MAXR][4];
    __shared__ unsigned long long tick[MAXR], start[MAXR];
    __shared__ float clear[MAXR];
    __shared__ unsigned char bits[MAXR];
    const int tid = threadIdx.x, R = q.R, base = blockIdx.x * R;

    if (tid < R) {
        const int a = base + tid;
        footprint(q, pose_in[a], c_in[tid]);
        footprint(q, pose_out[a], c_out[tid]);
        bits[tid] = (unsigned char)robot_bits(flags[a], closed[a], meta_in[a].y);
        tick[tid] = PACK_NONE;
        start[tid] = PACK_NONE;
    }

    // clearance: warp w takes robots w, w + 8, ...; float4 loads when the row is 16-byte aligned
    const int lane = tid & 31;
    for (int r = tid >> 5; r < R; r += SAFETY_WARPS) {
        const float *row = obs + (size_t)(base + r) * q.beams;
        float m = INFINITY;
        int k0 = 0;
        if (((uintptr_t)row & 15) == 0) {
            const float4 *row4 = reinterpret_cast<const float4 *>(row);
            for (int k = lane; k < q.beams >> 2; k += 32) {
                const float4 v = __ldg(row4 + k);
                m = fminf(fminf(m, fminf(v.x, v.y)), fminf(v.z, v.w));
            }
            k0 = q.beams & ~3;
        }
        for (int k = k0 + lane; k < q.beams; k += 32) m = fminf(m, __ldg(row + k));
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) clear[r] = clearance_metres(q, m);
    }
    __syncthreads();

    // separation: the R (R - 1) / 2 unordered pairs a < b over the CTA's threads, each computed once for both robots
    const int npairs = R * (R - 1) / 2;
    for (int p = tid; p < npairs; p += SAFETY_THREADS) {
        int a = 0, rest = p;
        while (rest >= R - 1 - a) {
            rest -= R - 1 - a;
            ++a;
        }
        const int b = a + 1 + rest, ba = bits[a], bb = bits[b];
        if (needs_out(ba, bb)) {
            const float s = separation(c_out[a], c_out[b]);
            if ((ba & ROBOT_TRACKED) && !(ba & ROBOT_RESPAWNED)) atomicMin(&tick[a], pack_sep(s, b));
            if ((bb & ROBOT_TRACKED) && !(bb & ROBOT_RESPAWNED)) atomicMin(&tick[b], pack_sep(s, a));
        }
        if (needs_in(ba, bb)) {
            const float s = separation(c_in[a], c_in[b]);
            if ((ba & ROBOT_TRACKED) && (ba & ROBOT_RESPAWNED)) atomicMin(&tick[a], pack_sep(s, b));
            if ((bb & ROBOT_TRACKED) && (bb & ROBOT_RESPAWNED)) atomicMin(&tick[b], pack_sep(s, a));
            if ((ba & ROBOT_TRACKED) && (ba & ROBOT_CRASHED)) atomicMin(&start[a], pack_sep(s, b));
            if ((bb & ROBOT_TRACKED) && (bb & ROBOT_CRASHED)) atomicMin(&start[b], pack_sep(s, a));
        }
    }
    __syncthreads();

    if (tid < R) {
        const int a = base + tid;
        const int32_t c = count[a];
        fold(q, flags[a], bits[tid], tick[tid], start[tid], clear[tid], c, min_sep + a, min_clear + a, last_clear + a,
             near + a, partner + a, records + (size_t)a * q.episodes + (c < q.episodes ? c : 0));
    }
}

// ------------------------------------------------------------------------------------------------ reduction
// float64 arithmetic without contraction, so that host, device and numpy round alike
__host__ __device__ __forceinline__ double d_add(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ double d_mul(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// Partials of world w, layout RLCA_SAFETY_* of include/rlca.h.  `split`: only the agents whose (mask != 0) equals
// `want` count.  erec are the tracker's records (result code in .x), srec this file's.
__host__ __device__ inline void safety_reduce_world(int R, int episodes, const float4 *srec, const float4 *erec,
                                                    const int32_t *count, int w, const uint8_t *mask, bool split,
                                                    bool want, double *out)
{
    double s[RLCA_SAFETY_NPARTIALS];
    for (int k = 0; k < RLCA_SAFETY_NPARTIALS; ++k) s[k] = 0.0;
    s[RLCA_SAFETY_MIN_SEPARATION] = (double)INFINITY;
    const auto inc = [&s](int k, double v) { s[k] = d_add(s[k], v); };
    for (int r = 0; r < R; ++r) {
        const int a = w * R + r;
        if (split && (mask[a] != 0) != want) continue;
        const int c = count[a];
        const int nrec = c < episodes ? c : episodes;
        for (int i = 0; i < nrec; ++i) {
            const float4 rec = srec[(size_t)a * episodes + i];
            const int packed = (int)rec.w, cause = packed & 3, hit = ((packed >> 8) & 0xff) - 1;
            const double sep = (double)rec.x, clr = (double)rec.y, nr = (double)rec.z;
            if (sep < s[RLCA_SAFETY_MIN_SEPARATION]) s[RLCA_SAFETY_MIN_SEPARATION] = sep;
            if (cause == 1) inc(RLCA_SAFETY_CRASH_STATIC, 1.0);
            if (cause == 2) {
                inc(RLCA_SAFETY_CRASH_ROBOT, 1.0);
                if (packed & 4) inc(RLCA_SAFETY_CRASH_BOTH_IN_RANGE, 1.0);
                if (mask && hit >= 0 && mask[w * R + hit] != 0) inc(RLCA_SAFETY_CRASH_INTO_MASKED, 1.0);
            }
            if ((int)erec[(size_t)a * episodes + i].x != 1) continue;
            inc(RLCA_SAFETY_REACHED, 1.0);
            if (rec.x < INFINITY) {
                inc(RLCA_SAFETY_REACHED_SEPARATION, 1.0);
                inc(RLCA_SAFETY_SUM_SEPARATION, sep);
                inc(RLCA_SAFETY_SUM_SEPARATION + 1, d_mul(sep, sep));
            }
            if (rec.y < INFINITY) {
                inc(RLCA_SAFETY_REACHED_CLEARANCE, 1.0);
                inc(RLCA_SAFETY_SUM_CLEARANCE, clr);
                inc(RLCA_SAFETY_SUM_CLEARANCE + 1, d_mul(clr, clr));
            }
            if (rec.z > 0.0f) inc(RLCA_SAFETY_NEAR_EPISODES, 1.0);
            inc(RLCA_SAFETY_SUM_NEAR_TICKS, nr);
        }
    }
    for (int k = 0; k < RLCA_SAFETY_NPARTIALS; ++k) out[k] = s[k];
}

// One thread per world, or per (world, role) with a mask: row 0 the agents with mask 0, row 1 the others.
__global__ void __launch_bounds__(REDUCE_THREADS) rlca_safety_reduce_kernel(int R, int episodes, const float4 *srec,
                                                                            const float4 *erec, const int32_t *count,
                                                                            const uint8_t *mask, int world_begin,
                                                                            int world_count, double *partials)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, rows = mask ? 2 : 1;
    if (i >= rows * world_count) return;
    safety_reduce_world(R, episodes, srec, erec, count, world_begin + i / rows, mask, mask != nullptr, i % rows,
                        partials + (size_t)i * RLCA_SAFETY_NPARTIALS);
}

// ------------------------------------------------------------------------------------------------ entries
static int safety_args(const rlca_env_config *cfg, const rlca_safety_params *p, int32_t episodes, SafetyParams &q)
{
    if (!cfg || !p) return rlca_set_err(RLCA_ERR_INVALID, "safety: cfg or params is NULL");
    if (cfg->robots_per_world < 1 || cfg->robots_per_world > RLCA_MAX_ROBOTS_PER_WORLD || cfg->num_worlds < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "safety: robots_per_world must be in 1..64 and num_worlds >= 1");
    if (cfg->beams < 1) return rlca_set_err(RLCA_ERR_INVALID, "safety: cfg has no beams");
    if (episodes < 1) return rlca_set_err(RLCA_ERR_INVALID, "safety: episodes must be >= 1");
    if (!(p->near_dist >= 0.0f && p->near_dist < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "safety: near_dist must be finite and >= 0");
    if (!(cfg->half_len > 0.0f && cfg->half_len < INFINITY && cfg->half_wid > 0.0f && cfg->half_wid < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID, "safety: cfg needs finite half_len > 0 and half_wid > 0");
    q.half_len = cfg->half_len;
    q.half_wid = cfg->half_wid;
    q.range_max = cfg->range_max;
    q.near_dist = p->near_dist;
    // two footprints that share a cell are at most sqrt(2) cells apart, and a footprint point moves at most
    // dt (v_max + |w| r_c) in a tick
    const float r_c = sqrtf(cfg->half_len * cfg->half_len + cfg->half_wid * cfg->half_wid);
    const float w_abs = fmaxf(fabsf(cfg->w_min), fabsf(cfg->w_max));
    q.contact = 1.41421356f * cfg->resolution + 2.0f * cfg->dt * (cfg->v_max + w_abs * r_c);
    q.R = cfg->robots_per_world;
    q.beams = cfg->beams;
    q.episodes = episodes;
    return RLCA_OK;
}

static int check_range(const rlca_env_config *cfg, int32_t world_begin, int32_t world_count)
{
    if (world_begin < 0 || world_count < 1 || world_begin > cfg->num_worlds - world_count)
        return rlca_set_err(RLCA_ERR_INVALID, "safety: world range outside the shard");
    return RLCA_OK;
}

extern "C" int rlca_safety_contact_host(const rlca_env_config *cfg, float *contact)
{
    const rlca_safety_params p = {0.0f};
    SafetyParams q;
    int rc = safety_args(cfg, &p, 1, q);
    if (rc) return rc;
    if (!contact) return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_contact_host: contact is NULL");
    *contact = q.contact;
    return RLCA_OK;
}

extern "C" int rlca_safety_separation_host(const rlca_env_config *cfg, const float *pose_a_host,
                                           const float *pose_b_host, int32_t n, float *separation_host)
{
    const rlca_safety_params p = {0.0f};
    SafetyParams q;
    int rc = safety_args(cfg, &p, 1, q);
    if (rc) return rc;
    if (!pose_a_host || !pose_b_host || !separation_host || n < 0)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_separation_host: a buffer is NULL or n < 0");
    for (int i = 0; i < n; ++i) {
        float2 A[4], B[4];
        footprint(q, reinterpret_cast<const float4 *>(pose_a_host)[i], A);
        footprint(q, reinterpret_cast<const float4 *>(pose_b_host)[i], B);
        separation_host[i] = separation(A, B);
    }
    return RLCA_OK;
}

extern "C" int rlca_safety_track(const rlca_env_config *cfg, const rlca_safety_params *params,
                                 const rlca_env_state *state_in, const rlca_env_state *state_out,
                                 const rlca_step_io *io, const rlca_eval_state *ev, const rlca_safety_state *ss,
                                 void *stream)
{
    SafetyParams q;
    int rc = safety_args(cfg, params, ss ? ss->episodes : 0, q);
    if (rc) return rc;
    if (!state_in || !state_out || !io || !ev || !ss)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_track: state, io, eval state or safety state is NULL");
    if (ev->episodes != ss->episodes)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_track: the tracker holds a different number of episodes");
    if (!state_in->pose_dev || !state_in->meta_dev || !state_out->pose_dev || !io->flags_dev || !io->obs_dev ||
        !ev->closed_dev || !ev->count_dev || !ss->min_sep_dev || !ss->min_clear_dev || !ss->last_clear_dev ||
        !ss->near_dev || !ss->partner_dev || !ss->records_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_track: a buffer is NULL");
    rlca_safety_track_kernel<<<cfg->num_worlds, SAFETY_THREADS, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const float4 *>(state_in->pose_dev), reinterpret_cast<const int4 *>(state_in->meta_dev),
        reinterpret_cast<const float4 *>(state_out->pose_dev), reinterpret_cast<const uchar4 *>(io->flags_dev),
        io->obs_dev, ev->closed_dev, ev->count_dev, ss->min_sep_dev, ss->min_clear_dev, ss->last_clear_dev,
        ss->near_dev, ss->partner_dev, reinterpret_cast<float4 *>(ss->records_dev));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_safety_track_host(const rlca_env_config *cfg, const rlca_safety_params *params,
                                      const float *pose_in_host, const int32_t *meta_in_host,
                                      const float *pose_out_host, const uint8_t *flags_host, const float *obs_host,
                                      const int32_t *closed_host, const int32_t *count_host, int32_t episodes,
                                      float *min_sep_host, float *min_clear_host, float *last_clear_host,
                                      int32_t *near_host, int32_t *partner_host, float *records_host)
{
    SafetyParams q;
    int rc = safety_args(cfg, params, episodes, q);
    if (rc) return rc;
    if (!pose_in_host || !meta_in_host || !pose_out_host || !flags_host || !obs_host || !closed_host || !count_host ||
        !min_sep_host || !min_clear_host || !last_clear_host || !near_host || !partner_host || !records_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_track_host: a buffer is NULL");
    const float4 *pose_in = reinterpret_cast<const float4 *>(pose_in_host);
    const float4 *pose_out = reinterpret_cast<const float4 *>(pose_out_host);
    const int4 *meta_in = reinterpret_cast<const int4 *>(meta_in_host);
    const uchar4 *flags = reinterpret_cast<const uchar4 *>(flags_host);
    float4 *records = reinterpret_cast<float4 *>(records_host);
    const int R = q.R;
    for (int w = 0; w < cfg->num_worlds; ++w) {
        const int base = w * R;
        float2 c_in[MAXR][4], c_out[MAXR][4];
        unsigned long long tick[MAXR], start[MAXR];
        float clear[MAXR];
        int bits[MAXR];
        for (int r = 0; r < R; ++r) {
            const int a = base + r;
            footprint(q, pose_in[a], c_in[r]);
            footprint(q, pose_out[a], c_out[r]);
            bits[r] = robot_bits(flags[a], closed_host[a], meta_in[a].y);
            tick[r] = start[r] = PACK_NONE;
            float m = INFINITY;
            for (int k = 0; k < q.beams; ++k) m = fminf(m, obs_host[(size_t)a * q.beams + k]);
            clear[r] = clearance_metres(q, m);
        }
        const auto lower = [](unsigned long long &dst, unsigned long long v) { if (v < dst) dst = v; };
        for (int a = 0; a < R; ++a)
            for (int b = a + 1; b < R; ++b) {
                const int ba = bits[a], bb = bits[b];
                if (needs_out(ba, bb)) {
                    const float s = separation(c_out[a], c_out[b]);
                    if ((ba & ROBOT_TRACKED) && !(ba & ROBOT_RESPAWNED)) lower(tick[a], pack_sep(s, b));
                    if ((bb & ROBOT_TRACKED) && !(bb & ROBOT_RESPAWNED)) lower(tick[b], pack_sep(s, a));
                }
                if (needs_in(ba, bb)) {
                    const float s = separation(c_in[a], c_in[b]);
                    if ((ba & ROBOT_TRACKED) && (ba & ROBOT_RESPAWNED)) lower(tick[a], pack_sep(s, b));
                    if ((bb & ROBOT_TRACKED) && (bb & ROBOT_RESPAWNED)) lower(tick[b], pack_sep(s, a));
                    if ((ba & ROBOT_TRACKED) && (ba & ROBOT_CRASHED)) lower(start[a], pack_sep(s, b));
                    if ((bb & ROBOT_TRACKED) && (bb & ROBOT_CRASHED)) lower(start[b], pack_sep(s, a));
                }
            }
        for (int r = 0; r < R; ++r) {
            const int a = base + r;
            const int32_t c = count_host[a];
            fold(q, flags[a], bits[r], tick[r], start[r], clear[r], c, min_sep_host + a, min_clear_host + a,
                 last_clear_host + a, near_host + a, partner_host + a,
                 records + (size_t)a * episodes + (c < episodes ? c : 0));
        }
    }
    return RLCA_OK;
}

extern "C" int rlca_safety_reduce(const rlca_env_config *cfg, const rlca_safety_state *ss, const rlca_eval_state *ev,
                                  const uint8_t *role_mask_dev, int32_t world_begin, int32_t world_count,
                                  double *partials_dev, void *stream)
{
    const rlca_safety_params p = {0.0f};
    SafetyParams q;
    int rc = safety_args(cfg, &p, ss ? ss->episodes : 0, q);
    if (rc) return rc;
    if ((rc = check_range(cfg, world_begin, world_count))) return rc;
    if (!ev) return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_reduce: eval state is NULL");
    if (ev->episodes != ss->episodes)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_reduce: the tracker holds a different number of episodes");
    if (!ss->records_dev || !ev->records_dev || !ev->count_dev || !partials_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_reduce: a buffer is NULL");
    const int threads = (role_mask_dev ? 2 : 1) * world_count;
    rlca_safety_reduce_kernel<<<(threads + REDUCE_THREADS - 1) / REDUCE_THREADS, REDUCE_THREADS, 0,
                                (cudaStream_t)stream>>>(
        q.R, q.episodes, reinterpret_cast<const float4 *>(ss->records_dev),
        reinterpret_cast<const float4 *>(ev->records_dev), ev->count_dev, role_mask_dev, world_begin, world_count,
        partials_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_safety_reduce_host(const rlca_env_config *cfg, const float *safety_records_host,
                                       const float *eval_records_host, const int32_t *count_host,
                                       const uint8_t *role_mask_host, int32_t episodes, int32_t world_begin,
                                       int32_t world_count, double *partials_host)
{
    const rlca_safety_params p = {0.0f};
    SafetyParams q;
    int rc = safety_args(cfg, &p, episodes, q);
    if (rc) return rc;
    if ((rc = check_range(cfg, world_begin, world_count))) return rc;
    if (!safety_records_host || !eval_records_host || !count_host || !partials_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_safety_reduce_host: a buffer is NULL");
    const int rows = role_mask_host ? 2 : 1;
    for (int i = 0; i < rows * world_count; ++i)
        safety_reduce_world(q.R, episodes, reinterpret_cast<const float4 *>(safety_records_host),
                            reinterpret_cast<const float4 *>(eval_records_host), count_host, world_begin + i / rows,
                            role_mask_host, role_mask_host != nullptr, i % rows,
                            partials_host + (size_t)i * RLCA_SAFETY_NPARTIALS);
    return RLCA_OK;
}
