// rlca_eval.cu — episode records and evaluation metrics on the device (sm_90a), C ABI in include/rlca.h.
//
// rlca_eval_track runs after each rlca_env_step and turns the tick's flags / eplog into one record per ended episode:
// result code, ticks, path length and straight-line start -> goal distance.  The path is the polyline through the
// robot's poses.  The one segment the poses cannot give is that of a tick that re-spawned the robot (auto_reset 1 or 2:
// the final pose was overwritten inside the tick); by the integration contract (DESIGN.md §4) such a tick moved it
// |v_clip| * dt along its old heading, or 0 when the move was reverted (crashed).
//
// rlca_eval_reduce sums the records of each world in float64, in a fixed order (agent, then record), one thread per
// world and no atomics, so a world's partials do not depend on the launch or on how the worlds are sharded.  The same
// per-world function runs on the host in rlca_eval_reduce_host, which the CPU tests check against numpy.
// rlca_eval_reduce_split runs it twice per world, once per role of an agent mask (DESIGN.md §9h).
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define EVAL_THREADS 128

__host__ __device__ __forceinline__ double d_hypot(double dx, double dy)
{
    return sqrt(d_add(d_mul(dx, dx), d_mul(dy, dy)));      // sqrt is correctly rounded on both sides
}

__global__ void __launch_bounds__(EVAL_THREADS) eval_track_kernel(
    int n, int episodes, float dt, float v_min, float v_max, const float4 *__restrict__ pose_in,
    const int4 *__restrict__ meta_in, const float4 *__restrict__ pose_out, const int4 *__restrict__ meta_out,
    const float2 *__restrict__ action, const uchar4 *__restrict__ flags, const float4 *__restrict__ eplog,
    double *__restrict__ path, int32_t *__restrict__ count, int32_t *__restrict__ closed, int32_t *__restrict__ open,
    float4 *__restrict__ records)
{
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n) return;
    const uchar4 fl = flags[a];                 // done, crashed, result, was_reset
    const int ep = meta_in[a].y;                // the episode this tick ran in
    int cl = closed[a];
    double len = path[a];
    if (cl != ep) {
        double seg;
        if (fl.w) {
            // re-spawned inside the tick: the command the tick used (only a live robot ends and re-spawns in one tick),
            // clipped as rlca_physics_kernel clips it
            float v = action[a].x;
            if (!(fabsf(v) <= 3.0e38f)) v = 0.0f;
            v = fminf(fmaxf(v, v_min), v_max);
            seg = fl.y ? 0.0 : d_mul(fabs((double)v), (double)dt);
        } else {
            const float4 p0 = pose_in[a], p1 = pose_out[a];
            seg = d_hypot((double)p1.x - (double)p0.x, (double)p1.y - (double)p0.y);
        }
        len = d_add(len, seg);
        if (fl.z != 0) {                        // the episode ended: eplog holds its row
            const int c = count[a];
            if (c < episodes) {
                const float4 e0 = eplog[2 * a], e1 = eplog[2 * a + 1];   // goal x, y, return, steps | init x, y, result, ep
                const float straight = (float)d_hypot((double)e0.x - (double)e1.x, (double)e0.y - (double)e1.y);
                records[(size_t)a * episodes + c] = make_float4(e1.z, e0.w, (float)len, straight);
            }
            count[a] = c + 1;
            cl = ep;
            closed[a] = cl;
            len = 0.0;
        }
    }
    if (fl.w) len = 0.0;                        // a new episode starts at the spawn pose
    path[a] = len;
    open[a] = cl != meta_out[a].y;
}

// Partials of world w (agents w*R .. w*R+R-1), layout RLCA_EVAL_* of include/rlca.h.  With a mask, only the agents
// whose (mask[a] != 0) equals `want` count.
__host__ __device__ inline void reduce_world(int R, int episodes, double dt, double v_max, double goal_radius,
                                             const float4 *records, const int32_t *count, const int32_t *open, int w,
                                             const uint8_t *mask, bool want, double *out)
{
    double s[RLCA_EVAL_NPARTIALS];
    for (int k = 0; k < RLCA_EVAL_NPARTIALS; ++k) s[k] = 0.0;
    for (int r = 0; r < R; ++r) {
        const int a = w * R + r;
        if (mask && (mask[a] != 0) != want) continue;
        const int c = count[a];
        const int nrec = c < episodes ? c : episodes;
        if (c < episodes && open[a]) s[RLCA_EVAL_UNFINISHED] = d_add(s[RLCA_EVAL_UNFINISHED], 1.0);
        for (int i = 0; i < nrec; ++i) {
            const float4 rec = records[(size_t)a * episodes + i];
            const int result = (int)rec.x;
            if (result == 2) { s[RLCA_EVAL_CRASHED] = d_add(s[RLCA_EVAL_CRASHED], 1.0); continue; }
            if (result == 3) { s[RLCA_EVAL_TIMED_OUT] = d_add(s[RLCA_EVAL_TIMED_OUT], 1.0); continue; }
            if (result != 1) continue;
            const double T = d_mul((double)rec.y, dt);
            const double len = (double)rec.z, D = (double)rec.w;
            const double Lr = d_add(D, -goal_radius);
            const double L = Lr > 0.0 ? Lr : 0.0;
            const double m[4] = {T, d_add(T, -(L / v_max)), d_add(len, -L), len / T};
            s[RLCA_EVAL_REACHED] = d_add(s[RLCA_EVAL_REACHED], 1.0);
            for (int k = 0; k < 4; ++k) {
                s[RLCA_EVAL_SUM_TIME + 2 * k] = d_add(s[RLCA_EVAL_SUM_TIME + 2 * k], m[k]);
                s[RLCA_EVAL_SUM_TIME + 2 * k + 1] = d_add(s[RLCA_EVAL_SUM_TIME + 2 * k + 1], d_mul(m[k], m[k]));
            }
            s[RLCA_EVAL_SUM_STRAIGHT] = d_add(s[RLCA_EVAL_SUM_STRAIGHT], D);
            s[RLCA_EVAL_SUM_PATH] = d_add(s[RLCA_EVAL_SUM_PATH], len);
        }
    }
    for (int k = 0; k < RLCA_EVAL_NPARTIALS; ++k) out[k] = s[k];
}

__global__ void __launch_bounds__(EVAL_THREADS) eval_reduce_kernel(int R, int episodes, double dt, double v_max,
                                                                    double goal_radius, const float4 *records,
                                                                    const int32_t *count, const int32_t *open,
                                                                    int world_begin, int world_count, double *partials)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= world_count) return;
    reduce_world(R, episodes, dt, v_max, goal_radius, records, count, open, world_begin + i, nullptr, false,
                 partials + (size_t)i * RLCA_EVAL_NPARTIALS);
}

// One thread per (world, row): row 0 the agents with mask 0, row 1 the others.
__global__ void __launch_bounds__(EVAL_THREADS) eval_reduce_split_kernel(int R, int episodes, double dt, double v_max,
                                                                          double goal_radius, const float4 *records,
                                                                          const int32_t *count, const int32_t *open,
                                                                          const uint8_t *mask, int world_begin,
                                                                          int world_count, double *partials)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * world_count) return;
    reduce_world(R, episodes, dt, v_max, goal_radius, records, count, open, world_begin + (i >> 1), mask, i & 1,
                 partials + (size_t)i * RLCA_EVAL_NPARTIALS);
}

static int check_cfg(const rlca_env_config *cfg, int32_t episodes)
{
    if (!cfg) return rlca_set_err(RLCA_ERR_INVALID, "cfg is NULL");
    if (int rc = rlca_check_robots(cfg, "eval")) return rc;
    if (episodes < 1) return rlca_set_err(RLCA_ERR_INVALID, "episodes must be >= 1");
    if (!(cfg->dt > 0.0f) || !(cfg->v_max > 0.0f)) return rlca_set_err(RLCA_ERR_INVALID, "cfg needs dt > 0 and v_max > 0");
    return RLCA_OK;
}

extern "C" int rlca_eval_track(const rlca_env_config *cfg, const rlca_env_state *state_in,
                               const rlca_env_state *state_out, const rlca_step_io *io, const rlca_eval_state *ev,
                               void *stream)
{
    int rc = check_cfg(cfg, ev ? ev->episodes : 0);
    if (rc) return rc;
    if (!state_in || !state_out || !io || !ev) return rlca_set_err(RLCA_ERR_INVALID, "state/io/eval state is NULL");
    if (!state_in->pose_dev || !state_in->meta_dev || !state_out->pose_dev || !state_out->meta_dev || !io->action_dev ||
        !io->flags_dev || !io->eplog_dev || !ev->path_dev || !ev->count_dev || !ev->closed_dev || !ev->open_dev ||
        !ev->records_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_eval_track: a buffer is NULL");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    eval_track_kernel<<<(n + EVAL_THREADS - 1) / EVAL_THREADS, EVAL_THREADS, 0, (cudaStream_t)stream>>>(
        n, ev->episodes, cfg->dt, cfg->v_min, cfg->v_max, reinterpret_cast<const float4 *>(state_in->pose_dev),
        reinterpret_cast<const int4 *>(state_in->meta_dev), reinterpret_cast<const float4 *>(state_out->pose_dev),
        reinterpret_cast<const int4 *>(state_out->meta_dev), reinterpret_cast<const float2 *>(io->action_dev),
        reinterpret_cast<const uchar4 *>(io->flags_dev), reinterpret_cast<const float4 *>(io->eplog_dev), ev->path_dev,
        ev->count_dev, ev->closed_dev, ev->open_dev, reinterpret_cast<float4 *>(ev->records_dev));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_eval_reduce(const rlca_env_config *cfg, const rlca_eval_state *ev, int32_t world_begin,
                                int32_t world_count, double *partials_dev, void *stream)
{
    int rc = check_cfg(cfg, ev ? ev->episodes : 0);
    if (rc) return rc;
    if ((rc = rlca_check_world_range(cfg, world_begin, world_count, "eval"))) return rc;
    if (!ev->count_dev || !ev->open_dev || !ev->records_dev || !partials_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_eval_reduce: a buffer is NULL");
    eval_reduce_kernel<<<(world_count + EVAL_THREADS - 1) / EVAL_THREADS, EVAL_THREADS, 0, (cudaStream_t)stream>>>(
        cfg->robots_per_world, ev->episodes, (double)cfg->dt, (double)cfg->v_max, (double)cfg->goal_radius,
        reinterpret_cast<const float4 *>(ev->records_dev), ev->count_dev, ev->open_dev, world_begin, world_count,
        partials_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_eval_reduce_host(const rlca_env_config *cfg, const float *records_host, const int32_t *count_host,
                                     const int32_t *open_host, int32_t episodes, int32_t world_begin,
                                     int32_t world_count, double *partials_host)
{
    int rc = check_cfg(cfg, episodes);
    if (rc) return rc;
    if ((rc = rlca_check_world_range(cfg, world_begin, world_count, "eval"))) return rc;
    if (!records_host || !count_host || !open_host || !partials_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_eval_reduce_host: a buffer is NULL");
    for (int i = 0; i < world_count; ++i)
        reduce_world(cfg->robots_per_world, episodes, (double)cfg->dt, (double)cfg->v_max, (double)cfg->goal_radius,
                     reinterpret_cast<const float4 *>(records_host), count_host, open_host, world_begin + i, nullptr,
                     false, partials_host + (size_t)i * RLCA_EVAL_NPARTIALS);
    return RLCA_OK;
}

extern "C" int rlca_eval_reduce_split(const rlca_env_config *cfg, const rlca_eval_state *ev, const uint8_t *mask_dev,
                                      int32_t world_begin, int32_t world_count, double *partials_dev, void *stream)
{
    int rc = check_cfg(cfg, ev ? ev->episodes : 0);
    if (rc) return rc;
    if ((rc = rlca_check_world_range(cfg, world_begin, world_count, "eval"))) return rc;
    if (!ev->count_dev || !ev->open_dev || !ev->records_dev || !mask_dev || !partials_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_eval_reduce_split: a buffer is NULL");
    eval_reduce_split_kernel<<<(2 * world_count + EVAL_THREADS - 1) / EVAL_THREADS, EVAL_THREADS, 0,
                               (cudaStream_t)stream>>>(
        cfg->robots_per_world, ev->episodes, (double)cfg->dt, (double)cfg->v_max, (double)cfg->goal_radius,
        reinterpret_cast<const float4 *>(ev->records_dev), ev->count_dev, ev->open_dev, mask_dev, world_begin,
        world_count, partials_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_eval_reduce_split_host(const rlca_env_config *cfg, const float *records_host,
                                           const int32_t *count_host, const int32_t *open_host,
                                           const uint8_t *mask_host, int32_t episodes, int32_t world_begin,
                                           int32_t world_count, double *partials_host)
{
    int rc = check_cfg(cfg, episodes);
    if (rc) return rc;
    if ((rc = rlca_check_world_range(cfg, world_begin, world_count, "eval"))) return rc;
    if (!records_host || !count_host || !open_host || !mask_host || !partials_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_eval_reduce_split_host: a buffer is NULL");
    for (int i = 0; i < 2 * world_count; ++i)
        reduce_world(cfg->robots_per_world, episodes, (double)cfg->dt, (double)cfg->v_max, (double)cfg->goal_radius,
                     reinterpret_cast<const float4 *>(records_host), count_host, open_host, world_begin + (i >> 1),
                     mask_host, i & 1, partials_host + (size_t)i * RLCA_EVAL_NPARTIALS);
    return RLCA_OK;
}
