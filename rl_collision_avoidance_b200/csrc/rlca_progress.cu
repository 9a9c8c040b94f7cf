// rlca_progress.cu — why robots time out or never finish (sm_90a), C ABI in include/rlca.h, DESIGN.md §9o.
//
// rlca_progress_track runs after each rlca_env_step and before that tick's rlca_eval_track.  Per robot and folded tick
// (a tick of a tracked episode that did not re-spawn the robot) it takes the distance to the goal the tick computed,
// the centre displacement and the heading change, and whether another robot of the world stands within block_dist,
// and folds them into the running episode: closest distance, ticks since the last progress_dist of progress, the run
// of still ticks and their total, rotation, robot near.  The episode boundaries are the tracker's (closed !=
// meta_in.y, record on flags.z != 0), read from its state and never written here.  A time-out gets its cause from the
// running state: frozen (still for `window` ticks), stalled (no progress for `window` ticks) or slow, + 4 with a robot
// near.
//
// One CTA per world, its robots' centres in shared memory.  Every function the kernel calls is __host__ __device__ and
// the file is built without FMA contraction on either side, so rlca_progress_track_host (serial loops over the same
// functions) equals the kernel bit for bit.  rlca_progress_reduce sums a world's records in float64 in
// agent-then-record order, one thread per world (and role), as rlca_eval_reduce does.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define PROGRESS_THREADS RLCA_MAX_ROBOTS_PER_WORLD
#define REDUCE_THREADS 128
#define MAXR RLCA_MAX_ROBOTS_PER_WORLD

struct ProgressParams {
    float progress_dist, still_dist, block_dist;
    int window, R, episodes;
};

// Is another robot's centre of the world strictly within block_dist of robot r's?  c: the world's R centres.
__host__ __device__ __forceinline__ bool robot_near(const ProgressParams &q, const float2 *c, int r)
{
    const float2 me = c[r];
    bool near = false;
    for (int j = 0; j < q.R; ++j) {
        const float dx = c[j].x - me.x, dy = c[j].y - me.y;
        near |= j != r && sqrtf(dx * dx + dy * dy) < q.block_dist;
    }
    return near;
}

// cause of an episode from its state: 1 frozen, 2 stalled, 3 slow, + 4 robot near.  n: since, run, still, ticks.
__host__ __device__ __forceinline__ int classify(const ProgressParams &q, int4 n, float near)
{
    return (n.y >= q.window ? 1 : n.x >= q.window ? 2 : 3) | (near != 0.0f ? 4 : 0);
}

// The running episode of one robot, folded with one tick; the record goes into the tracker's next slot.
// f: closest, ref, rotation, near; n: since, run, still, ticks.
__host__ __device__ __forceinline__ void fold(const ProgressParams &q, uchar4 fl, bool tracked, float4 p0, float4 p1,
                                              bool near_now, int32_t count, float4 *running, int4 *counters,
                                              float4 *record, uint8_t *cause)
{
    float4 f = *running;
    int4 n = *counters;
    bool restart = fl.w != 0;                  // a re-spawn: state_out already holds the next episode
    if (tracked) {
        if (!fl.w) {
            const float d = p1.w;
            const float dx = p1.x - p0.x, dy = p1.y - p0.y;
            const float s = sqrtf(dx * dx + dy * dy);
            if (n.w == 0) {
                f.x = d;
                f.y = d;
                n.x = 0;
            } else {
                f.x = fminf(f.x, d);
                if (d <= f.y - q.progress_dist) {
                    f.y = d;
                    n.x = 0;
                } else {
                    n.x += 1;
                }
            }
            if (s < q.still_dist) {
                n.y += 1;
                n.z += 1;
            } else {
                n.y = 0;
            }
            f.z += fabsf(dev_normalize(p1.z - p0.z));
            f.w = near_now ? 1.0f : 0.0f;
            n.w += 1;
        }
        if (fl.z != 0) {
            if (count < q.episodes) {
                *record = make_float4(f.x, f.z, (float)n.z, (float)n.w);
                *cause = (uint8_t)(fl.z == 3 ? classify(q, n, f.w) : 0);
            }
            restart = true;                     // the episode is over: start afresh
        }
    }
    if (restart) {
        f = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        n = make_int4(0, 0, 0, 0);
    }
    *running = f;
    *counters = n;
}

__global__ void __launch_bounds__(PROGRESS_THREADS) rlca_progress_track_kernel(
    ProgressParams q, const float4 *__restrict__ pose_in, const int4 *__restrict__ meta_in,
    const float4 *__restrict__ pose_out, const uchar4 *__restrict__ flags, const int32_t *__restrict__ closed,
    const int32_t *__restrict__ count, float4 *__restrict__ running, int4 *__restrict__ counters,
    float4 *__restrict__ records, uint8_t *__restrict__ causes)
{
    __shared__ float2 centre[MAXR];
    const int r = threadIdx.x, R = q.R, a = blockIdx.x * R + r;
    float4 p1 = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (r < R) {
        p1 = pose_out[a];
        centre[r] = make_float2(p1.x, p1.y);
    }
    __syncthreads();
    if (r >= R) return;
    const uchar4 fl = flags[a];
    const bool tracked = closed[a] != meta_in[a].y;
    const bool near_now = tracked && !fl.w && robot_near(q, centre, r);
    const int32_t c = count[a];
    const size_t slot = (size_t)a * q.episodes + (c < q.episodes ? c : 0);
    fold(q, fl, tracked, pose_in[a], p1, near_now, c, running + a, counters + a, records + slot, causes + slot);
}

// ------------------------------------------------------------------------------------------------ reduction
// the seven columns of one group (time-outs at base 0, unfinished episodes at base 7) for one episode.  The cause
// columns add 1 or 0 (exact either way), so that every index is a constant and the partials stay in registers.
__host__ __device__ __forceinline__ void tally(double *s, int base, int cause, float closest, bool folded)
{
    const int k = cause & 3;
    s[base] = d_add(s[base], k == 1 ? 1.0 : 0.0);
    s[base + 1] = d_add(s[base + 1], k == 2 ? 1.0 : 0.0);
    s[base + 2] = d_add(s[base + 2], k == 3 ? 1.0 : 0.0);
    s[base + 3] = d_add(s[base + 3], (cause & 4) ? 1.0 : 0.0);
    if (folded) {
        const double d = (double)closest;
        s[base + 4] = d_add(s[base + 4], 1.0);
        s[base + 5] = d_add(s[base + 5], d);
        s[base + 6] = d_add(s[base + 6], d_mul(d, d));
    }
}

// Partials of world w, layout RLCA_PROGRESS_* of include/rlca.h.  `split`: only the agents whose (mask != 0) equals
// `want` count.  erec, count, open are the tracker's; prec, causes, running, counters this file's.
__host__ __device__ inline void progress_reduce_world(const ProgressParams &q, const float4 *prec, const uint8_t *causes,
                                                      const float4 *running, const int4 *counters, const float4 *erec,
                                                      const int32_t *count, const int32_t *open, int w,
                                                      const uint8_t *mask, bool split, bool want, double *out)
{
    double s[RLCA_PROGRESS_NPARTIALS];
#pragma unroll
    for (int k = 0; k < RLCA_PROGRESS_NPARTIALS; ++k) s[k] = 0.0;
    const int E = q.episodes;
    for (int r = 0; r < q.R; ++r) {
        const int a = w * q.R + r;
        if (split && (mask[a] != 0) != want) continue;
        const int c = count[a];
        const int nrec = c < E ? c : E;
        for (int i = 0; i < nrec; ++i) {
            const size_t k = (size_t)a * E + i;
            const float4 rec = prec[k];
            const int result = (int)erec[k].x;
            s[RLCA_PROGRESS_SUM_STILL_TICKS] = d_add(s[RLCA_PROGRESS_SUM_STILL_TICKS], (double)rec.z);
            s[RLCA_PROGRESS_SUM_TICKS] = d_add(s[RLCA_PROGRESS_SUM_TICKS], (double)rec.w);
            if (result == 3) tally(s, RLCA_PROGRESS_TIMEOUT_FROZEN, causes[k], rec.x, rec.w > 0.0f);
            if (result != 1) continue;
            const double rot = (double)rec.y;
            s[RLCA_PROGRESS_REACHED] = d_add(s[RLCA_PROGRESS_REACHED], 1.0);
            s[RLCA_PROGRESS_SUM_ROTATION] = d_add(s[RLCA_PROGRESS_SUM_ROTATION], rot);
            s[RLCA_PROGRESS_SUM_ROTATION_SQ] = d_add(s[RLCA_PROGRESS_SUM_ROTATION_SQ], d_mul(rot, rot));
        }
        if (c < E && open[a]) {
            const float4 f = running[a];
            const int4 n = counters[a];
            tally(s, RLCA_PROGRESS_UNFINISHED_FROZEN, classify(q, n, f.w), f.x, n.w > 0);
        }
    }
#pragma unroll
    for (int k = 0; k < RLCA_PROGRESS_NPARTIALS; ++k) out[k] = s[k];
}

// One thread per world, or per (world, role) with a mask: row 0 the agents with mask 0, row 1 the others.
__global__ void __launch_bounds__(REDUCE_THREADS) rlca_progress_reduce_kernel(
    ProgressParams q, const float4 *prec, const uint8_t *causes, const float4 *running, const int4 *counters,
    const float4 *erec, const int32_t *count, const int32_t *open, const uint8_t *mask, int world_begin,
    int world_count, double *partials)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, rows = mask ? 2 : 1;
    if (i >= rows * world_count) return;
    progress_reduce_world(q, prec, causes, running, counters, erec, count, open, world_begin + i / rows, mask,
                          mask != nullptr, i % rows, partials + (size_t)i * RLCA_PROGRESS_NPARTIALS);
}

// ------------------------------------------------------------------------------------------------ entries
static int progress_args(const rlca_env_config *cfg, const rlca_progress_params *p, int32_t episodes,
                         ProgressParams &q)
{
    if (!cfg || !p) return rlca_set_err(RLCA_ERR_INVALID, "progress: cfg or params is NULL");
    if (int rc = rlca_check_robots(cfg, "progress")) return rc;
    if (episodes < 1) return rlca_set_err(RLCA_ERR_INVALID, "progress: episodes must be >= 1");
    if (p->window < 1) return rlca_set_err(RLCA_ERR_INVALID, "progress: window must be >= 1");
    if (!finite_nonneg(p->progress_dist) || !finite_nonneg(p->still_dist) || !finite_nonneg(p->block_dist))
        return rlca_set_err(RLCA_ERR_INVALID,
                            "progress: progress_dist, still_dist and block_dist must be finite and >= 0");
    q.progress_dist = p->progress_dist;
    q.still_dist = p->still_dist;
    q.block_dist = p->block_dist;
    q.window = p->window;
    q.R = cfg->robots_per_world;
    q.episodes = episodes;
    return RLCA_OK;
}

extern "C" int rlca_progress_track(const rlca_env_config *cfg, const rlca_progress_params *params,
                                   const rlca_env_state *state_in, const rlca_env_state *state_out,
                                   const rlca_step_io *io, const rlca_eval_state *ev, const rlca_progress_state *ps,
                                   void *stream)
{
    ProgressParams q;
    int rc = progress_args(cfg, params, ps ? ps->episodes : 0, q);
    if (rc) return rc;
    if (!state_in || !state_out || !io || !ev || !ps)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_track: state, io, eval state or progress state is NULL");
    if (ev->episodes != ps->episodes)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_track: the tracker holds a different number of episodes");
    if (!state_in->pose_dev || !state_in->meta_dev || !state_out->pose_dev || !io->flags_dev || !ev->closed_dev ||
        !ev->count_dev || !ps->running_dev || !ps->counters_dev || !ps->records_dev || !ps->causes_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_track: a buffer is NULL");
    const int threads = q.R > 32 ? 64 : 32;
    rlca_progress_track_kernel<<<cfg->num_worlds, threads, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const float4 *>(state_in->pose_dev), reinterpret_cast<const int4 *>(state_in->meta_dev),
        reinterpret_cast<const float4 *>(state_out->pose_dev), reinterpret_cast<const uchar4 *>(io->flags_dev),
        ev->closed_dev, ev->count_dev, reinterpret_cast<float4 *>(ps->running_dev),
        reinterpret_cast<int4 *>(ps->counters_dev), reinterpret_cast<float4 *>(ps->records_dev), ps->causes_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_progress_track_host(const rlca_env_config *cfg, const rlca_progress_params *params,
                                        const float *pose_in_host, const int32_t *meta_in_host,
                                        const float *pose_out_host, const uint8_t *flags_host,
                                        const int32_t *closed_host, const int32_t *count_host, int32_t episodes,
                                        float *running_host, int32_t *counters_host, float *records_host,
                                        uint8_t *causes_host)
{
    ProgressParams q;
    int rc = progress_args(cfg, params, episodes, q);
    if (rc) return rc;
    if (!pose_in_host || !meta_in_host || !pose_out_host || !flags_host || !closed_host || !count_host ||
        !running_host || !counters_host || !records_host || !causes_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_track_host: a buffer is NULL");
    const float4 *pose_in = reinterpret_cast<const float4 *>(pose_in_host);
    const float4 *pose_out = reinterpret_cast<const float4 *>(pose_out_host);
    const int4 *meta_in = reinterpret_cast<const int4 *>(meta_in_host);
    const uchar4 *flags = reinterpret_cast<const uchar4 *>(flags_host);
    float4 *running = reinterpret_cast<float4 *>(running_host);
    int4 *counters = reinterpret_cast<int4 *>(counters_host);
    float4 *records = reinterpret_cast<float4 *>(records_host);
    const int R = q.R;
    for (int w = 0; w < cfg->num_worlds; ++w) {
        float2 centre[MAXR];
        for (int r = 0; r < R; ++r) centre[r] = make_float2(pose_out[w * R + r].x, pose_out[w * R + r].y);
        for (int r = 0; r < R; ++r) {
            const int a = w * R + r;
            const uchar4 fl = flags[a];
            const bool tracked = closed_host[a] != meta_in[a].y;
            const bool near_now = tracked && !fl.w && robot_near(q, centre, r);
            const int32_t c = count_host[a];
            const size_t slot = (size_t)a * episodes + (c < episodes ? c : 0);
            fold(q, fl, tracked, pose_in[a], pose_out[a], near_now, c, running + a, counters + a, records + slot,
                 causes_host + slot);
        }
    }
    return RLCA_OK;
}

extern "C" int rlca_progress_reduce(const rlca_env_config *cfg, const rlca_progress_params *params,
                                    const rlca_progress_state *ps, const rlca_eval_state *ev,
                                    const uint8_t *role_mask_dev, int32_t world_begin, int32_t world_count,
                                    double *partials_dev, void *stream)
{
    ProgressParams q;
    int rc = progress_args(cfg, params, ps ? ps->episodes : 0, q);
    if (rc) return rc;
    if ((rc = rlca_check_world_range(cfg, world_begin, world_count, "progress"))) return rc;
    if (!ev) return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_reduce: eval state is NULL");
    if (ev->episodes != ps->episodes)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_reduce: the tracker holds a different number of episodes");
    if (!ps->records_dev || !ps->causes_dev || !ps->running_dev || !ps->counters_dev || !ev->records_dev ||
        !ev->count_dev || !ev->open_dev || !partials_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_reduce: a buffer is NULL");
    const int threads = (role_mask_dev ? 2 : 1) * world_count;
    rlca_progress_reduce_kernel<<<(threads + REDUCE_THREADS - 1) / REDUCE_THREADS, REDUCE_THREADS, 0,
                                  (cudaStream_t)stream>>>(
        q, reinterpret_cast<const float4 *>(ps->records_dev), ps->causes_dev,
        reinterpret_cast<const float4 *>(ps->running_dev), reinterpret_cast<const int4 *>(ps->counters_dev),
        reinterpret_cast<const float4 *>(ev->records_dev), ev->count_dev, ev->open_dev, role_mask_dev, world_begin,
        world_count, partials_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_progress_reduce_host(const rlca_env_config *cfg, const rlca_progress_params *params,
                                         const float *progress_records_host, const uint8_t *causes_host,
                                         const float *running_host, const int32_t *counters_host,
                                         const float *eval_records_host, const int32_t *count_host,
                                         const int32_t *open_host, const uint8_t *role_mask_host, int32_t episodes,
                                         int32_t world_begin, int32_t world_count, double *partials_host)
{
    ProgressParams q;
    int rc = progress_args(cfg, params, episodes, q);
    if (rc) return rc;
    if ((rc = rlca_check_world_range(cfg, world_begin, world_count, "progress"))) return rc;
    if (!progress_records_host || !causes_host || !running_host || !counters_host || !eval_records_host ||
        !count_host || !open_host || !partials_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_progress_reduce_host: a buffer is NULL");
    const int rows = role_mask_host ? 2 : 1;
    for (int i = 0; i < rows * world_count; ++i)
        progress_reduce_world(q, reinterpret_cast<const float4 *>(progress_records_host), causes_host,
                              reinterpret_cast<const float4 *>(running_host),
                              reinterpret_cast<const int4 *>(counters_host),
                              reinterpret_cast<const float4 *>(eval_records_host), count_host, open_host,
                              world_begin + i / rows, role_mask_host, role_mask_host != nullptr, i % rows,
                              partials_host + (size_t)i * RLCA_PROGRESS_NPARTIALS);
    return RLCA_OK;
}
