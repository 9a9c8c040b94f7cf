// rlca_layout.cu — random start / goal layouts for evaluation and training (sm_90a), C ABI in include/rlca.h,
// DESIGN.md §9i and §9k, the same sampler in the arenas of a generated obstacle map (§9v), and the arena curriculum's
// weighted arena draw, per-arena tally and weight update (§9z), at the end of the file.
//
// rlca_layout_random writes a layout into an env state in place, once before an episode: for world w (global index
// cfg.world_offset + w) and robots r = 0 .. R-1 in order, the start is the first try k < max_reject whose draw,
// uniform in the square [-side/2, side/2]^2, is at least `separation` from the starts placed so far; the goal the
// first try whose draw is at least `min_travel` from this start and `separation` from the goals placed so far; the
// heading one draw u * 2 pi, wrapped as the env's spawn wraps it.  Draws use the env's Philox keys with agent =
// global world * R + r, episode 0, draw k and the layout purposes of rlca_common.cuh (start, goal, heading), so a
// world's layout depends only on (seed, global world, R, parameters, max_reject).
//
// Distances are compared squared, and draws and tests use plain float32 + - x (this file is compiled with
// -fmad=false on the device and -ffp-contract=off on the host), so rlca_layout_random_host gives the same bits.
//
// One warp per world, the world's placed starts and goals in shared memory: lane l evaluates try base + l and the
// lowest accepting lane wins (ballot, shuffle) in rounds of 32 tries — the order of the host's sequential loop.  When
// no try of the budget is accepted the world's rows are left untouched and status[w] = 1 + r.
//
// Training (§9k) runs two launches after each tick of an env with auto_reset 0: rlca_layout_respawn parks the robots
// whose episode ended and re-lays a world whose robots have all ended theirs with the same sampler at episode
// meta.y + 1 (so a re-layout never repeats an earlier layout's draws), and, after rlca_env_observe on the new state,
// rlca_stack_refresh makes the re-laid robots' scan FIFOs three copies of their new scan, as the tick does after an
// in-tick re-spawn.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include <vector>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define LAYOUT_THREADS 256
#define LAYOUT_WARPS (LAYOUT_THREADS / 32)

namespace {

struct LayoutConsts {
    uint64_t seed;
    uint32_t agent0;         // global agent index of the world's robot 0
    float side, sep2, travel2;
    uint32_t episode;        // Philox episode counter of the draws: 0 for rlca_layout_random, meta.y + 1 for a re-layout
};

// try k of robot r's start or goal: uniform in the square, one rounding per coordinate
// ((u - 0.5) is exact for the 24-bit uniforms)
__host__ __device__ __forceinline__ void layout_draw(const LayoutConsts &c, uint32_t r, uint32_t k, uint32_t purpose,
                                                     float &x, float &y)
{
    float u[4];
    dev_rand4(c.seed, c.agent0 + r, c.episode, k, purpose, u);
    x = (u[0] - 0.5f) * c.side;
    y = (u[1] - 0.5f) * c.side;
}

__host__ __device__ __forceinline__ float layout_heading(const LayoutConsts &c, uint32_t r)
{
    float u[4];
    dev_rand4(c.seed, c.agent0 + r, c.episode, 0u, PURPOSE_LAYOUT_HEADING, u);
    return dev_normalize(u[0] * 6.28318548202514648438f);
}

__host__ __device__ __forceinline__ float dist2(float ax, float ay, float bx, float by)
{
    const float dx = ax - bx, dy = ay - by;
    return dx * dx + dy * dy;
}

// a start draw at least `separation` from the starts px/py[0 .. r-1]
__host__ __device__ __forceinline__ bool start_ok(const LayoutConsts &c, const float *px, const float *py, int r,
                                                  float x, float y)
{
    for (int j = 0; j < r; ++j)
        if (!(dist2(x, y, px[j], py[j]) >= c.sep2)) return false;
    return true;
}

// a goal draw at least `min_travel` from the start (sx, sy) and `separation` from the goals qx/qy[0 .. r-1]
__host__ __device__ __forceinline__ bool goal_ok(const LayoutConsts &c, const float *qx, const float *qy, int r,
                                                 float sx, float sy, float x, float y)
{
    if (!(dist2(x, y, sx, sy) >= c.travel2)) return false;
    return start_ok(c, qx, qy, r, x, y);
}

// The records of one placed robot, as apply_spawn (rlca_env.cu) writes a spawn without starting an episode.
__host__ __device__ __forceinline__ void layout_apply(int pre_distance_zero, float x, float y, float th, float gx,
                                                      float gy, float4 &pose, float4 &goal, float4 &acc)
{
    pose.x = x; pose.y = y; pose.z = th;
    goal.x = gx; goal.y = gy;
    const float ddx = gx - x, ddy = gy - y;
    const float d0 = sqrtf(fmaf(ddx, ddx, ddy * ddy));
    pose.w = pre_distance_zero ? 0.0f : d0;
    acc.z = x; acc.w = y;
}

struct LayoutSmem {
    float sx[RLCA_MAX_ROBOTS_PER_WORLD], sy[RLCA_MAX_ROBOTS_PER_WORLD];
    float gx[RLCA_MAX_ROBOTS_PER_WORLD], gy[RLCA_MAX_ROBOTS_PER_WORLD];
};

// The draws of the square (rlca_layout_random): try k of robot r at the start or goal purpose.
struct SquareDraw {
    __host__ __device__ __forceinline__ void operator()(const LayoutConsts &c, uint32_t r, uint32_t k, uint32_t purpose,
                                                        float &x, float &y) const
    {
        layout_draw(c, r, k, purpose, x, y);
    }
};

// The first accepted try of robot r (start or goal purpose) by the whole warp; false when none of the budget is.
template <class Draw>
__device__ __forceinline__ bool warp_place(const Draw &draw, const LayoutConsts &c, const LayoutSmem &s, int r,
                                           uint32_t purpose, int max_reject, int lane, float &ox, float &oy)
{
    for (int base = 0; base < max_reject; base += 32) {
        const int k = base + lane;
        float x = 0.f, y = 0.f;
        bool ok = false;
        if (k < max_reject) {
            draw(c, (uint32_t)r, (uint32_t)k, purpose, x, y);
            ok = purpose == PURPOSE_LAYOUT_START ? start_ok(c, s.sx, s.sy, r, x, y) : goal_ok(c, s.gx, s.gy, r, s.sx[r], s.sy[r], x, y);
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, ok);
        if (mask) {
            const int src = __ffs(mask) - 1;
            ox = __shfl_sync(0xffffffffu, x, src);
            oy = __shfl_sync(0xffffffffu, y, src);
            return true;
        }
    }
    return false;
}

// The starts and goals of robots 0 .. R-1 of one world into s by the whole warp: true, or false with *status = 1 + r
// when robot r found no accepted try (s then holds robots 0 .. r-1 only).  The loop of rlca_layout_random_kernel, which
// keeps it inline: written through this function its SASS is scheduled differently, though it computes the same.
template <class Draw>
__device__ __forceinline__ bool warp_layout(const Draw &draw, const LayoutConsts &c, LayoutSmem &s, int R,
                                            int max_reject, int lane, int32_t *status)
{
    for (int r = 0; r < R; ++r) {
        float x, y, gx, gy;
        if (!warp_place(draw, c, s, r, PURPOSE_LAYOUT_START, max_reject, lane, x, y)) {
            if (lane == 0) *status = 1 + r;
            return false;
        }
        if (lane == 0) { s.sx[r] = x; s.sy[r] = y; }
        __syncwarp();
        if (!warp_place(draw, c, s, r, PURPOSE_LAYOUT_GOAL, max_reject, lane, gx, gy)) {
            if (lane == 0) *status = 1 + r;
            return false;
        }
        if (lane == 0) { s.gx[r] = gx; s.gy[r] = gy; }
        __syncwarp();
    }
    return true;
}

// The same by one thread, trying in order: the host twins' loop.
template <class Draw>
inline int host_layout(const Draw &draw, const LayoutConsts &c, int R, int max_reject, float *sx, float *sy, float *gx,
                       float *gy)
{
    for (int r = 0; r < R; ++r) {
        int k = 0;
        for (; k < max_reject; ++k) {
            draw(c, (uint32_t)r, (uint32_t)k, PURPOSE_LAYOUT_START, sx[r], sy[r]);
            if (start_ok(c, sx, sy, r, sx[r], sy[r])) break;
        }
        if (k == max_reject) return 1 + r;
        for (k = 0; k < max_reject; ++k) {
            draw(c, (uint32_t)r, (uint32_t)k, PURPOSE_LAYOUT_GOAL, gx[r], gy[r]);
            if (goal_ok(c, gx, gy, r, sx[r], sy[r], gx[r], gy[r])) break;
        }
        if (k == max_reject) return 1 + r;
    }
    return 0;
}

__global__ void __launch_bounds__(LAYOUT_THREADS)
rlca_layout_random_kernel(int num_worlds, int R, int max_reject, int pre_distance_zero, int world_offset,
                          uint64_t seed, float side, float sep2, float travel2, float4 *__restrict__ pose,
                          float4 *__restrict__ goal, float4 *__restrict__ acc, int32_t *__restrict__ status)
{
    __shared__ LayoutSmem smem[LAYOUT_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * LAYOUT_WARPS + wib;
    if (w >= num_worlds) return;                     // warp-uniform
    LayoutSmem &s = smem[wib];
    const LayoutConsts c = { seed, (uint32_t)(world_offset + w) * (uint32_t)R, side, sep2, travel2, 0u };
    for (int r = 0; r < R; ++r) {
        float x, y, gx, gy;
        if (!warp_place(SquareDraw(), c, s, r, PURPOSE_LAYOUT_START, max_reject, lane, x, y)) {
            if (lane == 0) status[w] = 1 + r;
            return;
        }
        if (lane == 0) { s.sx[r] = x; s.sy[r] = y; }
        __syncwarp();
        if (!warp_place(SquareDraw(), c, s, r, PURPOSE_LAYOUT_GOAL, max_reject, lane, gx, gy)) {
            if (lane == 0) status[w] = 1 + r;
            return;
        }
        if (lane == 0) { s.gx[r] = gx; s.gy[r] = gy; }
        __syncwarp();
    }
    for (int r = lane; r < R; r += 32) {
        const size_t i = (size_t)w * R + r;
        float4 p = pose[i], g = goal[i], a = acc[i];
        layout_apply(pre_distance_zero, s.sx[r], s.sy[r], layout_heading(c, (uint32_t)r), s.gx[r], s.gy[r], p, g, a);
        pose[i] = p; goal[i] = g; acc[i] = a;
    }
    if (lane == 0) status[w] = 0;
}

// The records of one re-laid robot, as apply_spawn writes a spawn that starts episode e; its last command is zero.
__host__ __device__ __forceinline__ void relayout_apply(int pre_distance_zero, float x, float y, float th, float gx,
                                                        float gy, int e, float4 &pose, float4 &goal, float4 &acc,
                                                        int4 &meta)
{
    layout_apply(pre_distance_zero, x, y, th, gx, gy, pose, goal, acc);
    goal.z = 0.0f; goal.w = 0.0f;
    acc.x = 0.0f;
    meta.x = 1; meta.y = e; meta.w = 0;
}

// The sampler of the square: warp_layout with the square's draws.
struct SquareSampler {
    __device__ __forceinline__ bool operator()(const LayoutConsts &c, uint32_t /*world*/, LayoutSmem &s, int R,
                                               int max_reject, int lane, int32_t *status) const
    {
        return warp_layout(SquareDraw(), c, s, R, max_reject, lane, status);
    }
};

// One world of a re-layout launch, by its warp: park the latched robots (meta.w != 0) and re-lay the world when its
// robots are all latched, with `sampler` at episode meta.y + 1.
template <class Sampler>
__device__ __forceinline__ void respawn_world(const Sampler &sampler, LayoutSmem &s, int w, int lane, int R,
                                              int max_reject, int pre_distance_zero, int world_offset, uint64_t seed,
                                              float side, float sep2, float travel2, float4 *__restrict__ pose,
                                              float4 *__restrict__ goal, float4 *__restrict__ acc,
                                              int4 *__restrict__ meta, uint8_t *__restrict__ flags,
                                              uint8_t *__restrict__ live, int32_t *__restrict__ status)
{
    const size_t i0 = (size_t)w * R;
    // robots lane and lane + 32 (R <= 64)
    const bool l0 = lane < R && meta[i0 + lane].w != 0;
    const bool l1 = lane + 32 < R && meta[i0 + lane + 32].w != 0;
    const int latched = __popc(__ballot_sync(0xffffffffu, l0)) + __popc(__ballot_sync(0xffffffffu, l1));
    if (latched == R) {                              // warp-uniform
        const int e = meta[i0].y + 1;
        const LayoutConsts c = { seed, (uint32_t)(world_offset + w) * (uint32_t)R, side, sep2, travel2, (uint32_t)e };
        if (sampler(c, (uint32_t)(world_offset + w), s, R, max_reject, lane, status + w)) {
            for (int r = lane; r < R; r += 32) {
                const size_t i = i0 + r;
                float4 p = pose[i], g = goal[i], a = acc[i];
                int4 m = meta[i];
                relayout_apply(pre_distance_zero, s.sx[r], s.sy[r], layout_heading(c, (uint32_t)r), s.gx[r], s.gy[r],
                               e, p, g, a, m);
                pose[i] = p; goal[i] = g; acc[i] = a; meta[i] = m;
                flags[4 * i + 3] = 1;
                live[i] = 1;
            }
            if (lane == 0) status[w] = 0;
            return;
        }
    }
    for (int r = lane; r < R; r += 32) {
        const size_t i = i0 + r;
        const bool parked = (r < 32 ? l0 : l1);
        if (parked) {
            float4 g = goal[i];
            g.z = 0.0f; g.w = 0.0f;
            goal[i] = g;
        }
        live[i] = parked ? 0 : 1;
    }
    if (lane == 0 && latched != R) status[w] = 0;    // a failed re-layout keeps the status warp_layout wrote
}

// After a tick (auto_reset 0): park the latched robots (meta.w != 0) of every world and re-lay a world whose robots
// are all latched with the sampler of rlca_layout_random_kernel at episode meta.y + 1.  One warp per world.
__global__ void __launch_bounds__(LAYOUT_THREADS)
rlca_layout_respawn_kernel(int num_worlds, int R, int max_reject, int pre_distance_zero, int world_offset,
                           uint64_t seed, float side, float sep2, float travel2, float4 *__restrict__ pose,
                           float4 *__restrict__ goal, float4 *__restrict__ acc, int4 *__restrict__ meta,
                           uint8_t *__restrict__ flags, uint8_t *__restrict__ live, int32_t *__restrict__ status)
{
    __shared__ LayoutSmem smem[LAYOUT_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * LAYOUT_WARPS + wib;
    if (w >= num_worlds) return;                     // warp-uniform
    respawn_world(SquareSampler(), smem[wib], w, lane, R, max_reject, pre_distance_zero, world_offset, seed, side, sep2,
                  travel2, pose, goal, acc, meta, flags, live, status);
}

// ---------------------------------------------------------------------------------------------- arenas (§9v)
// Try k of robot r in one arena: a uniform cell of the arena's list, then a uniform point of that cell.
struct ArenaDraw {
    const int32_t *cells;    // the arena's cells, cx | cy << 16
    uint32_t n;              // and their count
    int ocx, ocy;
    float res;
    __host__ __device__ __forceinline__ void operator()(const LayoutConsts &c, uint32_t r, uint32_t k, uint32_t purpose,
                                                        float &x, float &y) const
    {
        float u[4];
        dev_rand4(c.seed, c.agent0 + r, c.episode, k, PURPOSE_ARENA | purpose, u);
        const uint64_t m = (uint64_t)(u[0] * 16777216.0f);          // exact: u[0] is a multiple of 2^-24
        const uint32_t cell = (uint32_t)cells[(m * n) >> 24];
        x = ((float)((int)(cell & 0xffffu) - ocx) + u[1]) * res;
        y = ((float)((int)(cell >> 16) - ocy) + u[2]) * res;
    }
};

struct ArenaArgs {
    const int32_t *cell_off, *cells;
    int T, pick, ocx, ocy;
    float res;
};

// The arena of global world `world` at the episode of c: pick 0 world mod T, pick 1 one draw keyed by robot 0.
__host__ __device__ __forceinline__ int arena_of(const LayoutConsts &c, const ArenaArgs &t, uint32_t world)
{
    if (t.pick == 0) return (int)(world % (uint32_t)t.T);
    float u[4];
    dev_rand4(c.seed, c.agent0, c.episode, 0u, PURPOSE_ARENA, u);
    return (int)(((uint64_t)(u[0] * 16777216.0f) * (uint32_t)t.T) >> 24);
}

// The draws of arena a.
__host__ __device__ __forceinline__ ArenaDraw arena_cells_draw(const ArenaArgs &t, int a)
{
    const int32_t off = t.cell_off[a];
    return ArenaDraw{ t.cells + off, (uint32_t)(t.cell_off[a + 1] - off), t.ocx, t.ocy, t.res };
}

__host__ __device__ __forceinline__ ArenaDraw arena_draw(const LayoutConsts &c, const ArenaArgs &t, uint32_t world)
{
    return arena_cells_draw(t, arena_of(c, t, world));
}

struct ArenaSampler {
    ArenaArgs t;
    __device__ __forceinline__ bool operator()(const LayoutConsts &c, uint32_t world, LayoutSmem &s, int R,
                                               int max_reject, int lane, int32_t *status) const
    {
        return warp_layout(arena_draw(c, t, world), c, s, R, max_reject, lane, status);
    }
};

__global__ void __launch_bounds__(LAYOUT_THREADS)
rlca_layout_arena_kernel(int num_worlds, int R, int max_reject, int pre_distance_zero, int world_offset, uint64_t seed,
                         float sep2, float travel2, ArenaArgs t, float4 *__restrict__ pose, float4 *__restrict__ goal,
                         float4 *__restrict__ acc, int32_t *__restrict__ status)
{
    __shared__ LayoutSmem smem[LAYOUT_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * LAYOUT_WARPS + wib;
    if (w >= num_worlds) return;                     // warp-uniform
    LayoutSmem &s = smem[wib];
    const LayoutConsts c = { seed, (uint32_t)(world_offset + w) * (uint32_t)R, 0.0f, sep2, travel2, 0u };
    if (!ArenaSampler{ t }(c, (uint32_t)(world_offset + w), s, R, max_reject, lane, status + w)) return;
    for (int r = lane; r < R; r += 32) {
        const size_t i = (size_t)w * R + r;
        float4 p = pose[i], g = goal[i], a = acc[i];
        layout_apply(pre_distance_zero, s.sx[r], s.sy[r], layout_heading(c, (uint32_t)r), s.gx[r], s.gy[r], p, g, a);
        pose[i] = p; goal[i] = g; acc[i] = a;
    }
    if (lane == 0) status[w] = 0;
}

__global__ void __launch_bounds__(LAYOUT_THREADS)
rlca_layout_arena_respawn_kernel(int num_worlds, int R, int max_reject, int pre_distance_zero, int world_offset,
                                 uint64_t seed, float sep2, float travel2, ArenaArgs t, float4 *__restrict__ pose,
                                 float4 *__restrict__ goal, float4 *__restrict__ acc, int4 *__restrict__ meta,
                                 uint8_t *__restrict__ flags, uint8_t *__restrict__ live, int32_t *__restrict__ status)
{
    __shared__ LayoutSmem smem[LAYOUT_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * LAYOUT_WARPS + wib;
    if (w >= num_worlds) return;                     // warp-uniform
    respawn_world(ArenaSampler{ t }, smem[wib], w, lane, R, max_reject, pre_distance_zero, world_offset, seed, 0.0f,
                  sep2, travel2, pose, goal, acc, meta, flags, live, status);
}

// The FIFO slot of a re-laid agent (flags.w set) becomes three copies of its scan, and its goal | speed row is
// replaced.  One warp per agent, coalesced 16-byte copies.
__global__ void __launch_bounds__(LAYOUT_THREADS)
rlca_stack_refresh_kernel(int n, int scan4, const uint8_t *__restrict__ flags, const float4 *__restrict__ obs,
                          const float4 *__restrict__ gs_src, float4 *__restrict__ stack, float4 *__restrict__ gs)
{
    const int a = blockIdx.x * LAYOUT_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (a >= n || flags[4 * (size_t)a + 3] == 0) return;          // warp-uniform
    const float4 *src = obs + (size_t)a * scan4;
    float4 *dst = stack + (size_t)a * 3 * scan4;
    for (int c = lane; c < scan4; c += 32) {
        const float4 v = src[c];
        dst[c] = v; dst[scan4 + c] = v; dst[2 * scan4 + c] = v;
    }
    if (lane == 0) gs[a] = gs_src[a];
}

// `square`: the params' side bounds the layout (rlca_layout_random / _respawn); an arena layout has no side.
int check_layout(const rlca_env_config *cfg, const rlca_layout_params *params, const char *who, bool square = true)
{
    if (!cfg || !params) return rlca_set_err(RLCA_ERR_INVALID, "%s: cfg or params is NULL", who);
    if (cfg->robots_per_world < 2 || cfg->robots_per_world > RLCA_MAX_ROBOTS_PER_WORLD)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: robots_per_world must be in [2, 64]", who);
    if (cfg->num_worlds < 1) return rlca_set_err(RLCA_ERR_INVALID, "%s: num_worlds must be >= 1", who);
    if (cfg->max_reject < 1) return rlca_set_err(RLCA_ERR_INVALID, "%s: max_reject must be >= 1", who);
    if (cfg->world_offset < 0) return rlca_set_err(RLCA_ERR_INVALID, "%s: world_offset must be >= 0", who);
    if (square) {
        const double side = params->side;
        if (!(side > 0.0 && side < INFINITY))
            return rlca_set_err(RLCA_ERR_INVALID, "%s: side must be finite and > 0", who);
        if (!(params->min_travel >= 0.0f && (double)params->min_travel <= side * sqrt(2.0)))
            return rlca_set_err(RLCA_ERR_INVALID, "%s: min_travel must be in [0, side * sqrt(2)]", who);
    } else if (!(params->min_travel >= 0.0f && params->min_travel < INFINITY)) {
        return rlca_set_err(RLCA_ERR_INVALID, "%s: min_travel must be finite and >= 0", who);
    }
    // two footprints whose centres are this far apart share no cell, whatever their headings
    const double rc = sqrt((double)cfg->half_len * cfg->half_len + (double)cfg->half_wid * cfg->half_wid);
    if (!(params->separation > 2.0 * (rc + sqrt(2.0) * (double)cfg->resolution) && params->separation < INFINITY))
        return rlca_set_err(RLCA_ERR_INVALID,
                            "%s: separation must be finite and > 2 (r_c + sqrt(2) resolution), r_c the footprint's "
                            "circumradius", who);
    return RLCA_OK;
}

LayoutConsts layout_consts(const rlca_env_config *cfg, const rlca_layout_params *params, int w, uint32_t episode)
{
    return { cfg->seed, (uint32_t)(cfg->world_offset + w) * (uint32_t)cfg->robots_per_world, params->side,
             params->separation * params->separation, params->min_travel * params->min_travel, episode };
}

// The checks of an arena layout's arguments that need no table contents: those the device entries make.
int check_arena(const rlca_env_config *cfg, const rlca_layout_params *params, const rlca_arena_tables *tables,
                int32_t pick, const char *who)
{
    int rc = check_layout(cfg, params, who, false);
    if (rc) return rc;
    if (!tables || !tables->cell_off || !tables->cells)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: tables, tables->cell_off or tables->cells is NULL", who);
    if (tables->num_arenas < 1) return rlca_set_err(RLCA_ERR_INVALID, "%s: tables->num_arenas must be >= 1", who);
    if (pick != 0 && pick != 1) return rlca_set_err(RLCA_ERR_INVALID, "%s: pick must be 0 (world) or 1 (draw)", who);
    return RLCA_OK;
}

// The table contents, from host memory: offsets from 0, strictly increasing (no empty arena), cells on the map.
int check_arena_cells(const rlca_env_config *cfg, const rlca_arena_tables *t, const char *who)
{
    if (t->cell_off[0] != 0) return rlca_set_err(RLCA_ERR_INVALID, "%s: tables->cell_off[0] must be 0", who);
    for (int a = 0; a < t->num_arenas; ++a) {
        if (t->cell_off[a + 1] == t->cell_off[a]) return rlca_set_err(RLCA_ERR_INVALID, "%s: an arena is empty", who);
        if (t->cell_off[a + 1] < t->cell_off[a])
            return rlca_set_err(RLCA_ERR_INVALID, "%s: tables->cell_off decreases", who);
    }
    for (int32_t i = 0; i < t->cell_off[t->num_arenas]; ++i) {
        const uint32_t cell = (uint32_t)t->cells[i];
        if ((int)(cell & 0xffffu) >= cfg->grid_w || (int)(cell >> 16) >= cfg->grid_h)
            return rlca_set_err(RLCA_ERR_INVALID, "%s: a cell lies outside the map", who);
    }
    return RLCA_OK;
}

ArenaArgs arena_args(const rlca_env_config *cfg, const rlca_arena_tables *t, int32_t pick)
{
    return { t->cell_off, t->cells, t->num_arenas, pick, cfg->origin_cx, cfg->origin_cy, cfg->resolution };
}

// ---------------------------------------------------------------------------------------------- curriculum (§9z)
// An arena drawn in proportion to integer weights w_a: pick 1's draw m = 2^24 u0 (agent g R, episode, draw 0, purpose
// 0xA0) and the arena a with cdf[a] <= (m cdf[T]) >> 24 < cdf[a + 1], cdf the exclusive prefix sum of w.  Equal weights
// W give floor(floor(m T W / 2^24) / W) = (m T) >> 24, pick 1's arena.  T < 2^20 and w <= 2^20 keep m cdf[T] < 2^64.
#define CURRICULUM_THREADS 1024
#define CURRICULUM_MAX_ARENAS (1 << 20)
#define CURRICULUM_ONE 1048576.0f                    // 2^20: the weight of score 1

__host__ __device__ __forceinline__ int weighted_arena(const LayoutConsts &c, const uint64_t *cdf, int T)
{
    float u[4];
    dev_rand4(c.seed, c.agent0, c.episode, 0u, PURPOSE_ARENA, u);
    const uint64_t target = ((uint64_t)(u[0] * 16777216.0f) * cdf[T]) >> 24;
    int lo = 0, hi = T;                              // the largest lo < T with cdf[lo] <= target
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (cdf[mid] <= target) lo = mid; else hi = mid;
    }
    return lo;
}

// The arena sampler with the weighted draw; world_arena[world - world_offset] records the arena of a layout that
// succeeded, and keeps the old arena when one fails.
struct WeightedArenaSampler {
    ArenaArgs t;
    const uint64_t *cdf;
    int32_t *world_arena;
    int world_offset;
    __device__ __forceinline__ bool operator()(const LayoutConsts &c, uint32_t world, LayoutSmem &s, int R,
                                               int max_reject, int lane, int32_t *status) const
    {
        const int a = weighted_arena(c, cdf, t.T);
        if (!warp_layout(arena_cells_draw(t, a), c, s, R, max_reject, lane, status)) return false;
        if (lane == 0) world_arena[(int)world - world_offset] = a;
        return true;
    }
};

// The ended rows of world w in this tick's flags (x != 0 and z != 0; success z == 1), rows with row_mask != 0 left
// out, added to pending[a] (episodes) and pending[T + a] (successes) of the world's arena a.  One integer atomic per
// counter per world, so the sums do not depend on the order of the worlds.
__device__ __forceinline__ void tally_world(int w, int lane, int R, int T, const uint8_t *__restrict__ flags,
                                            const uint8_t *__restrict__ row_mask,
                                            const int32_t *__restrict__ world_arena, int32_t *__restrict__ pending)
{
    const size_t i0 = (size_t)w * R;
    int ended = 0, reached = 0;
    for (int r = lane; r < 64; r += 32) {            // robots lane and lane + 32 (R <= 64), the loop warp-uniform
        bool e = false, s = false;
        if (r < R && !(row_mask && row_mask[i0 + r])) {
            const uint8_t fx = flags[4 * (i0 + r)], fz = flags[4 * (i0 + r) + 2];
            e = fx != 0 && fz != 0;
            s = e && fz == 1;
        }
        ended += __popc(__ballot_sync(0xffffffffu, e));
        reached += __popc(__ballot_sync(0xffffffffu, s));
    }
    if (lane == 0 && ended) {
        const int a = world_arena[w];
        if (a >= 0 && a < T) {
            atomicAdd(pending + a, ended);
            if (reached) atomicAdd(pending + T + a, reached);
        }
    }
}

__global__ void __launch_bounds__(LAYOUT_THREADS)
rlca_layout_arena_weighted_kernel(int num_worlds, int R, int max_reject, int pre_distance_zero, int world_offset,
                                  uint64_t seed, float sep2, float travel2, ArenaArgs t,
                                  const uint64_t *__restrict__ cdf, int32_t *__restrict__ world_arena,
                                  float4 *__restrict__ pose, float4 *__restrict__ goal, float4 *__restrict__ acc,
                                  int32_t *__restrict__ status)
{
    __shared__ LayoutSmem smem[LAYOUT_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * LAYOUT_WARPS + wib;
    if (w >= num_worlds) return;                     // warp-uniform
    LayoutSmem &s = smem[wib];
    const LayoutConsts c = { seed, (uint32_t)(world_offset + w) * (uint32_t)R, 0.0f, sep2, travel2, 0u };
    const WeightedArenaSampler sampler{ t, cdf, world_arena, world_offset };
    if (!sampler(c, (uint32_t)(world_offset + w), s, R, max_reject, lane, status + w)) return;
    for (int r = lane; r < R; r += 32) {
        const size_t i = (size_t)w * R + r;
        float4 p = pose[i], g = goal[i], a = acc[i];
        layout_apply(pre_distance_zero, s.sx[r], s.sy[r], layout_heading(c, (uint32_t)r), s.gx[r], s.gy[r], p, g, a);
        pose[i] = p; goal[i] = g; acc[i] = a;
    }
    if (lane == 0) status[w] = 0;
}

// After a tick (auto_reset 0): tally the tick's ended rows against each world's arena, then park and re-lay as
// rlca_layout_arena_respawn_kernel does, with the weighted arena draw.  One warp per world.
__global__ void __launch_bounds__(LAYOUT_THREADS)
rlca_layout_arena_weighted_respawn_kernel(int num_worlds, int R, int max_reject, int pre_distance_zero,
                                          int world_offset, uint64_t seed, float sep2, float travel2, ArenaArgs t,
                                          const uint64_t *__restrict__ cdf, int32_t *__restrict__ world_arena,
                                          int32_t *__restrict__ pending, const uint8_t *__restrict__ row_mask,
                                          float4 *__restrict__ pose, float4 *__restrict__ goal,
                                          float4 *__restrict__ acc, int4 *__restrict__ meta,
                                          uint8_t *__restrict__ flags, uint8_t *__restrict__ live,
                                          int32_t *__restrict__ status)
{
    __shared__ LayoutSmem smem[LAYOUT_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * LAYOUT_WARPS + wib;
    if (w >= num_worlds) return;                     // warp-uniform
    // lane 0 reads the world's arena here before its sampler writes a new one
    tally_world(w, lane, R, t.T, flags, row_mask, world_arena, pending);
    respawn_world(WeightedArenaSampler{ t, cdf, world_arena, world_offset }, smem[wib], w, lane, R, max_reject,
                  pre_distance_zero, world_offset, seed, 0.0f, sep2, travel2, pose, goal, acc, meta, flags, live,
                  status);
}

// Fold one update's counts into the decayed counts of arena a and return its weight, in float32 with one rounding
// per operation: E = decay E + e, S = decay S + s, p = (S + 1) / (E + 2), q = uniform + (1 - uniform) 4 p (1 - p),
// w = max(1, floor(2^20 q)).  q <= 1 whenever E, S >= 0; the clamp to 2^20 keeps the bound for any stored values.
__host__ __device__ __forceinline__ uint32_t curriculum_fold(float &E, float &S, int32_t e, int32_t s, float decay,
                                                             float uniform)
{
    E = decay * E + (float)e;
    S = decay * S + (float)s;
    const float p = (S + 1.0f) / (E + 2.0f);
    const float q = uniform + (1.0f - uniform) * (4.0f * p * (1.0f - p));
    const float v = q * CURRICULUM_ONE;
    return v >= CURRICULUM_ONE ? (uint32_t)CURRICULUM_ONE : v >= 1.0f ? (uint32_t)v : 1u;
}

// One CTA: every arena's fold, pending zeroed, and the exclusive prefix sum of the weights into cdf (cdf[T] the
// total), 1024 arenas per round with a carry.  Integer sums: the result does not depend on the thread order.
__global__ void __launch_bounds__(CURRICULUM_THREADS)
rlca_arena_curriculum_update_kernel(int T, float decay, float uniform, float *__restrict__ E, float *__restrict__ S,
                                    int32_t *__restrict__ pending, unsigned long long *__restrict__ cdf)
{
    __shared__ unsigned long long warp_sum[CURRICULUM_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long carry = 0;
    for (int base = 0; base < T; base += CURRICULUM_THREADS) {
        const int a = base + threadIdx.x;
        unsigned long long w = 0;
        if (a < T) {
            float e = E[a], s = S[a];
            w = curriculum_fold(e, s, pending[a], pending[T + a], decay, uniform);
            E[a] = e; S[a] = s;
            pending[a] = 0; pending[T + a] = 0;
        }
        unsigned long long x = w;                    // inclusive scan in the warp
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_sum[wid] = x;
        __syncthreads();
        if (wid == 0) {
            unsigned long long v = warp_sum[lane];
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned long long y = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= d) v += y;
            }
            warp_sum[lane] = v;
        }
        __syncthreads();
        if (a < T) cdf[a] = carry + (wid ? warp_sum[wid - 1] : 0ull) + x - w;
        carry += warp_sum[CURRICULUM_THREADS / 32 - 1];
        __syncthreads();                             // warp_sum is rewritten by the next round
    }
    if (threadIdx.x == 0) cdf[T] = carry;
}

int check_curriculum(const rlca_arena_curriculum *cur, const char *who)
{
    if (!cur || !cur->cdf || !cur->world_arena || !cur->pending || !cur->E || !cur->S)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: curriculum or one of its buffers is NULL", who);
    if (cur->num_arenas < 1 || cur->num_arenas >= CURRICULUM_MAX_ARENAS)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: curriculum->num_arenas must be in [1, 2^20)", who);
    return RLCA_OK;
}

// check_arena with pick 1 (the weighted draw replaces it), and a curriculum over the tables' arenas
int check_weighted(const rlca_env_config *cfg, const rlca_layout_params *params, const rlca_arena_tables *tables,
                   const rlca_arena_curriculum *cur, const char *who)
{
    int rc = check_arena(cfg, params, tables, 1, who);
    if (!rc) rc = check_curriculum(cur, who);
    if (rc) return rc;
    if (cur->num_arenas != tables->num_arenas)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: curriculum->num_arenas must equal tables->num_arenas", who);
    return RLCA_OK;
}

}  // namespace

extern "C" int rlca_layout_random(const rlca_env_config *cfg, const rlca_layout_params *params,
                                  const rlca_env_state *state, int32_t *status_dev, void *stream)
{
    int rc = check_layout(cfg, params, "rlca_layout_random");
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->acc_dev || !status_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_random: a state or status buffer is NULL");
    const LayoutConsts c = layout_consts(cfg, params, 0, 0u);
    const int ctas = (cfg->num_worlds + LAYOUT_WARPS - 1) / LAYOUT_WARPS;
    rlca_layout_random_kernel<<<ctas, LAYOUT_THREADS, 0, (cudaStream_t)stream>>>(
        cfg->num_worlds, cfg->robots_per_world, cfg->max_reject, cfg->pre_distance_zero, cfg->world_offset, c.seed,
        c.side, c.sep2, c.travel2, reinterpret_cast<float4 *>(state->pose_dev),
        reinterpret_cast<float4 *>(state->goal_dev), reinterpret_cast<float4 *>(state->acc_dev), status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

// The host twins' loops over the worlds: `draw_of(c, w)` gives world w's draws at the episode of c.
template <class DrawOf>
static void host_layout_worlds(const rlca_env_config *cfg, const rlca_layout_params *params, const DrawOf &draw_of,
                        float *pose_host, float *goal_host, float *acc_host, int32_t *status_host)
{
    const int R = cfg->robots_per_world;
    float4 *pose = reinterpret_cast<float4 *>(pose_host), *goal = reinterpret_cast<float4 *>(goal_host);
    float4 *acc = reinterpret_cast<float4 *>(acc_host);
    for (int w = 0; w < cfg->num_worlds; ++w) {
        const LayoutConsts c = layout_consts(cfg, params, w, 0u);
        float sx[RLCA_MAX_ROBOTS_PER_WORLD], sy[RLCA_MAX_ROBOTS_PER_WORLD];
        float gx[RLCA_MAX_ROBOTS_PER_WORLD], gy[RLCA_MAX_ROBOTS_PER_WORLD];
        const int failed = host_layout(draw_of(c, w), c, R, cfg->max_reject, sx, sy, gx, gy);
        status_host[w] = failed;
        if (failed) continue;
        for (int r = 0; r < R; ++r) {
            const size_t i = (size_t)w * R + r;
            layout_apply(cfg->pre_distance_zero, sx[r], sy[r], layout_heading(c, (uint32_t)r), gx[r], gy[r], pose[i],
                         goal[i], acc[i]);
        }
    }
}

template <class DrawOf>
static void host_respawn_worlds(const rlca_env_config *cfg, const rlca_layout_params *params, const DrawOf &draw_of,
                         float *pose_host, float *goal_host, float *acc_host, int32_t *meta_host, uint8_t *flags_host,
                         uint8_t *live_host, int32_t *status_host)
{
    const int R = cfg->robots_per_world;
    float4 *pose = reinterpret_cast<float4 *>(pose_host), *goal = reinterpret_cast<float4 *>(goal_host);
    float4 *acc = reinterpret_cast<float4 *>(acc_host);
    int4 *meta = reinterpret_cast<int4 *>(meta_host);
    for (int w = 0; w < cfg->num_worlds; ++w) {
        const size_t i0 = (size_t)w * R;
        int latched = 0;
        for (int r = 0; r < R; ++r) latched += meta[i0 + r].w != 0;
        int failed = 0;
        if (latched == R) {
            const int e = meta[i0].y + 1;
            const LayoutConsts c = layout_consts(cfg, params, w, (uint32_t)e);
            float sx[RLCA_MAX_ROBOTS_PER_WORLD], sy[RLCA_MAX_ROBOTS_PER_WORLD];
            float gx[RLCA_MAX_ROBOTS_PER_WORLD], gy[RLCA_MAX_ROBOTS_PER_WORLD];
            failed = host_layout(draw_of(c, w), c, R, cfg->max_reject, sx, sy, gx, gy);
            if (!failed) {
                for (int r = 0; r < R; ++r) {
                    const size_t i = i0 + r;
                    relayout_apply(cfg->pre_distance_zero, sx[r], sy[r], layout_heading(c, (uint32_t)r), gx[r], gy[r],
                                   e, pose[i], goal[i], acc[i], meta[i]);
                    flags_host[4 * i + 3] = 1;
                    live_host[i] = 1;
                }
                status_host[w] = 0;
                continue;
            }
        }
        for (int r = 0; r < R; ++r) {
            const size_t i = i0 + r;
            const bool parked = meta[i].w != 0;
            if (parked) { goal[i].z = 0.0f; goal[i].w = 0.0f; }
            live_host[i] = parked ? 0 : 1;
        }
        status_host[w] = failed;
    }
}

extern "C" int rlca_layout_random_host(const rlca_env_config *cfg, const rlca_layout_params *params, float *pose_host,
                                       float *goal_host, float *acc_host, int32_t *status_host)
{
    int rc = check_layout(cfg, params, "rlca_layout_random_host");
    if (rc) return rc;
    if (!pose_host || !goal_host || !acc_host || !status_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_random_host: a buffer is NULL");
    host_layout_worlds(cfg, params, [](const LayoutConsts &, int) { return SquareDraw(); }, pose_host, goal_host,
                       acc_host, status_host);
    return RLCA_OK;
}

static int check_respawn(const rlca_env_config *cfg, const rlca_layout_params *params, const char *who)
{
    int rc = check_layout(cfg, params, who);
    if (rc) return rc;
    if (cfg->auto_reset != 0) return rlca_set_err(RLCA_ERR_INVALID, "%s: cfg.auto_reset must be 0", who);
    return RLCA_OK;
}

extern "C" int rlca_layout_respawn(const rlca_env_config *cfg, const rlca_layout_params *params,
                                   const rlca_env_state *state, uint8_t *flags_dev, uint8_t *live_dev,
                                   int32_t *status_dev, void *stream)
{
    int rc = check_respawn(cfg, params, "rlca_layout_respawn");
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->acc_dev || !state->meta_dev || !flags_dev ||
        !live_dev || !status_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_respawn: a state, flags, live or status buffer is NULL");
    const LayoutConsts c = layout_consts(cfg, params, 0, 0u);
    const int ctas = (cfg->num_worlds + LAYOUT_WARPS - 1) / LAYOUT_WARPS;
    rlca_layout_respawn_kernel<<<ctas, LAYOUT_THREADS, 0, (cudaStream_t)stream>>>(
        cfg->num_worlds, cfg->robots_per_world, cfg->max_reject, cfg->pre_distance_zero, cfg->world_offset, c.seed,
        c.side, c.sep2, c.travel2, reinterpret_cast<float4 *>(state->pose_dev),
        reinterpret_cast<float4 *>(state->goal_dev), reinterpret_cast<float4 *>(state->acc_dev),
        reinterpret_cast<int4 *>(state->meta_dev), flags_dev, live_dev, status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_layout_respawn_host(const rlca_env_config *cfg, const rlca_layout_params *params, float *pose_host,
                                        float *goal_host, float *acc_host, int32_t *meta_host, uint8_t *flags_host,
                                        uint8_t *live_host, int32_t *status_host)
{
    int rc = check_respawn(cfg, params, "rlca_layout_respawn_host");
    if (rc) return rc;
    if (!pose_host || !goal_host || !acc_host || !meta_host || !flags_host || !live_host || !status_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_respawn_host: a buffer is NULL");
    host_respawn_worlds(cfg, params, [](const LayoutConsts &, int) { return SquareDraw(); }, pose_host, goal_host,
                        acc_host, meta_host, flags_host, live_host, status_host);
    return RLCA_OK;
}

extern "C" int rlca_stack_refresh(const rlca_env_config *cfg, const uint8_t *flags_dev, const float *obs_dev,
                                  const float *gs_src_dev, float *stack_dev, float *gs_dev, void *stream)
{
    if (!cfg) return rlca_set_err(RLCA_ERR_INVALID, "rlca_stack_refresh: cfg is NULL");
    if (int rc = rlca_check_robots(cfg, "rlca_stack_refresh")) return rc;
    if (cfg->beams < 1 || (3 * cfg->beams) % 4 != 0)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_stack_refresh: 3 * beams must be a multiple of 4");
    if (!flags_dev || !obs_dev || !gs_src_dev || !stack_dev || !gs_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_stack_refresh: a buffer is NULL");
    if (((uintptr_t)obs_dev | (uintptr_t)gs_src_dev | (uintptr_t)stack_dev | (uintptr_t)gs_dev) & 15)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_stack_refresh: misaligned buffer");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const int ctas = (n + LAYOUT_WARPS - 1) / LAYOUT_WARPS;
    rlca_stack_refresh_kernel<<<ctas, LAYOUT_THREADS, 0, (cudaStream_t)stream>>>(
        n, cfg->beams / 4, flags_dev, reinterpret_cast<const float4 *>(obs_dev),
        reinterpret_cast<const float4 *>(gs_src_dev), reinterpret_cast<float4 *>(stack_dev),
        reinterpret_cast<float4 *>(gs_dev));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

// ---------------------------------------------------------------------------------------------- arenas (§9v)
extern "C" int rlca_arena_tables_check(const rlca_env_config *cfg, const rlca_arena_tables *tables_host)
{
    if (!cfg) return rlca_set_err(RLCA_ERR_INVALID, "rlca_arena_tables_check: cfg is NULL");
    if (!tables_host || !tables_host->cell_off || !tables_host->cells)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_arena_tables_check: tables, cell_off or cells is NULL");
    if (tables_host->num_arenas < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_arena_tables_check: tables->num_arenas must be >= 1");
    return check_arena_cells(cfg, tables_host, "rlca_arena_tables_check");
}

extern "C" int rlca_layout_arena(const rlca_env_config *cfg, const rlca_layout_params *params,
                                 const rlca_arena_tables *tables, int32_t pick, const rlca_env_state *state,
                                 int32_t *status_dev, void *stream)
{
    int rc = check_arena(cfg, params, tables, pick, "rlca_layout_arena");
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->acc_dev || !status_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_arena: a state or status buffer is NULL");
    const LayoutConsts c = layout_consts(cfg, params, 0, 0u);
    const int ctas = (cfg->num_worlds + LAYOUT_WARPS - 1) / LAYOUT_WARPS;
    rlca_layout_arena_kernel<<<ctas, LAYOUT_THREADS, 0, (cudaStream_t)stream>>>(
        cfg->num_worlds, cfg->robots_per_world, cfg->max_reject, cfg->pre_distance_zero, cfg->world_offset, c.seed,
        c.sep2, c.travel2, arena_args(cfg, tables, pick), reinterpret_cast<float4 *>(state->pose_dev),
        reinterpret_cast<float4 *>(state->goal_dev), reinterpret_cast<float4 *>(state->acc_dev), status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_layout_arena_host(const rlca_env_config *cfg, const rlca_layout_params *params,
                                      const rlca_arena_tables *tables_host, int32_t pick, float *pose_host,
                                      float *goal_host, float *acc_host, int32_t *status_host)
{
    int rc = check_arena(cfg, params, tables_host, pick, "rlca_layout_arena_host");
    if (!rc) rc = check_arena_cells(cfg, tables_host, "rlca_layout_arena_host");
    if (rc) return rc;
    if (!pose_host || !goal_host || !acc_host || !status_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_arena_host: a buffer is NULL");
    const ArenaArgs t = arena_args(cfg, tables_host, pick);
    host_layout_worlds(cfg, params,
                       [&](const LayoutConsts &c, int w) { return arena_draw(c, t, (uint32_t)(cfg->world_offset + w)); },
                       pose_host, goal_host, acc_host, status_host);
    return RLCA_OK;
}

static int check_arena_respawn(const rlca_env_config *cfg, const rlca_layout_params *params,
                               const rlca_arena_tables *tables, int32_t pick, const char *who)
{
    int rc = check_arena(cfg, params, tables, pick, who);
    if (rc) return rc;
    if (cfg->auto_reset != 0) return rlca_set_err(RLCA_ERR_INVALID, "%s: cfg.auto_reset must be 0", who);
    return RLCA_OK;
}

extern "C" int rlca_layout_arena_respawn(const rlca_env_config *cfg, const rlca_layout_params *params,
                                         const rlca_arena_tables *tables, int32_t pick, const rlca_env_state *state,
                                         uint8_t *flags_dev, uint8_t *live_dev, int32_t *status_dev, void *stream)
{
    int rc = check_arena_respawn(cfg, params, tables, pick, "rlca_layout_arena_respawn");
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->acc_dev || !state->meta_dev || !flags_dev ||
        !live_dev || !status_dev)
        return rlca_set_err(RLCA_ERR_INVALID,
                            "rlca_layout_arena_respawn: a state, flags, live or status buffer is NULL");
    const LayoutConsts c = layout_consts(cfg, params, 0, 0u);
    const int ctas = (cfg->num_worlds + LAYOUT_WARPS - 1) / LAYOUT_WARPS;
    rlca_layout_arena_respawn_kernel<<<ctas, LAYOUT_THREADS, 0, (cudaStream_t)stream>>>(
        cfg->num_worlds, cfg->robots_per_world, cfg->max_reject, cfg->pre_distance_zero, cfg->world_offset, c.seed,
        c.sep2, c.travel2, arena_args(cfg, tables, pick), reinterpret_cast<float4 *>(state->pose_dev),
        reinterpret_cast<float4 *>(state->goal_dev), reinterpret_cast<float4 *>(state->acc_dev),
        reinterpret_cast<int4 *>(state->meta_dev), flags_dev, live_dev, status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_layout_arena_respawn_host(const rlca_env_config *cfg, const rlca_layout_params *params,
                                              const rlca_arena_tables *tables_host, int32_t pick, float *pose_host,
                                              float *goal_host, float *acc_host, int32_t *meta_host,
                                              uint8_t *flags_host, uint8_t *live_host, int32_t *status_host)
{
    int rc = check_arena_respawn(cfg, params, tables_host, pick, "rlca_layout_arena_respawn_host");
    if (!rc) rc = check_arena_cells(cfg, tables_host, "rlca_layout_arena_respawn_host");
    if (rc) return rc;
    if (!pose_host || !goal_host || !acc_host || !meta_host || !flags_host || !live_host || !status_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_arena_respawn_host: a buffer is NULL");
    const ArenaArgs t = arena_args(cfg, tables_host, pick);
    host_respawn_worlds(cfg, params,
                        [&](const LayoutConsts &c, int w) { return arena_draw(c, t, (uint32_t)(cfg->world_offset + w)); },
                        pose_host, goal_host, acc_host, meta_host, flags_host, live_host, status_host);
    return RLCA_OK;
}

// ---------------------------------------------------------------------------------------------- curriculum (§9z)
extern "C" int rlca_layout_arena_weighted(const rlca_env_config *cfg, const rlca_layout_params *params,
                                          const rlca_arena_tables *tables, const rlca_arena_curriculum *curriculum,
                                          const rlca_env_state *state, int32_t *status_dev, void *stream)
{
    int rc = check_weighted(cfg, params, tables, curriculum, "rlca_layout_arena_weighted");
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !state->acc_dev || !status_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_arena_weighted: a state or status buffer is NULL");
    const LayoutConsts c = layout_consts(cfg, params, 0, 0u);
    const int ctas = (cfg->num_worlds + LAYOUT_WARPS - 1) / LAYOUT_WARPS;
    rlca_layout_arena_weighted_kernel<<<ctas, LAYOUT_THREADS, 0, (cudaStream_t)stream>>>(
        cfg->num_worlds, cfg->robots_per_world, cfg->max_reject, cfg->pre_distance_zero, cfg->world_offset, c.seed,
        c.sep2, c.travel2, arena_args(cfg, tables, 1), curriculum->cdf, curriculum->world_arena,
        reinterpret_cast<float4 *>(state->pose_dev), reinterpret_cast<float4 *>(state->goal_dev),
        reinterpret_cast<float4 *>(state->acc_dev), status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_layout_arena_weighted_host(const rlca_env_config *cfg, const rlca_layout_params *params,
                                               const rlca_arena_tables *tables_host,
                                               const rlca_arena_curriculum *curriculum_host, float *pose_host,
                                               float *goal_host, float *acc_host, int32_t *status_host)
{
    int rc = check_weighted(cfg, params, tables_host, curriculum_host, "rlca_layout_arena_weighted_host");
    if (!rc) rc = check_arena_cells(cfg, tables_host, "rlca_layout_arena_weighted_host");
    if (rc) return rc;
    if (!pose_host || !goal_host || !acc_host || !status_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_layout_arena_weighted_host: a buffer is NULL");
    const ArenaArgs t = arena_args(cfg, tables_host, 1);
    const rlca_arena_curriculum &cur = *curriculum_host;
    std::vector<int> drawn(cfg->num_worlds, -1);
    host_layout_worlds(cfg, params,
                       [&](const LayoutConsts &c, int w) {
                           drawn[w] = weighted_arena(c, cur.cdf, t.T);
                           return arena_cells_draw(t, drawn[w]);
                       },
                       pose_host, goal_host, acc_host, status_host);
    for (int w = 0; w < cfg->num_worlds; ++w)
        if (status_host[w] == 0) cur.world_arena[w] = drawn[w];
    return RLCA_OK;
}

extern "C" int rlca_layout_arena_weighted_respawn(const rlca_env_config *cfg, const rlca_layout_params *params,
                                                  const rlca_arena_tables *tables,
                                                  const rlca_arena_curriculum *curriculum, const uint8_t *row_mask_dev,
                                                  const rlca_env_state *state, uint8_t *flags_dev, uint8_t *live_dev,
                                                  int32_t *status_dev, void *stream)
{
    const char *who = "rlca_layout_arena_weighted_respawn";
    int rc = check_weighted(cfg, params, tables, curriculum, who);
    if (rc) return rc;
    if (cfg->auto_reset != 0) return rlca_set_err(RLCA_ERR_INVALID, "%s: cfg.auto_reset must be 0", who);
    if (!state || !state->pose_dev || !state->goal_dev || !state->acc_dev || !state->meta_dev || !flags_dev ||
        !live_dev || !status_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: a state, flags, live or status buffer is NULL", who);
    const LayoutConsts c = layout_consts(cfg, params, 0, 0u);
    const int ctas = (cfg->num_worlds + LAYOUT_WARPS - 1) / LAYOUT_WARPS;
    rlca_layout_arena_weighted_respawn_kernel<<<ctas, LAYOUT_THREADS, 0, (cudaStream_t)stream>>>(
        cfg->num_worlds, cfg->robots_per_world, cfg->max_reject, cfg->pre_distance_zero, cfg->world_offset, c.seed,
        c.sep2, c.travel2, arena_args(cfg, tables, 1), curriculum->cdf, curriculum->world_arena, curriculum->pending,
        row_mask_dev, reinterpret_cast<float4 *>(state->pose_dev), reinterpret_cast<float4 *>(state->goal_dev),
        reinterpret_cast<float4 *>(state->acc_dev), reinterpret_cast<int4 *>(state->meta_dev), flags_dev, live_dev,
        status_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_layout_arena_weighted_respawn_host(const rlca_env_config *cfg, const rlca_layout_params *params,
                                                       const rlca_arena_tables *tables_host,
                                                       const rlca_arena_curriculum *curriculum_host,
                                                       const uint8_t *row_mask_host, float *pose_host,
                                                       float *goal_host, float *acc_host, int32_t *meta_host,
                                                       uint8_t *flags_host, uint8_t *live_host, int32_t *status_host)
{
    const char *who = "rlca_layout_arena_weighted_respawn_host";
    int rc = check_weighted(cfg, params, tables_host, curriculum_host, who);
    if (!rc) rc = check_arena_cells(cfg, tables_host, who);
    if (rc) return rc;
    if (cfg->auto_reset != 0) return rlca_set_err(RLCA_ERR_INVALID, "%s: cfg.auto_reset must be 0", who);
    if (!pose_host || !goal_host || !acc_host || !meta_host || !flags_host || !live_host || !status_host)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: a buffer is NULL", who);
    const ArenaArgs t = arena_args(cfg, tables_host, 1);
    const rlca_arena_curriculum &cur = *curriculum_host;
    const int R = cfg->robots_per_world, T = t.T;
    for (int w = 0; w < cfg->num_worlds; ++w) {                  // the tally, against the arenas before re-layout
        int ended = 0, reached = 0;
        for (int r = 0; r < R; ++r) {
            const size_t i = (size_t)w * R + r;
            if (row_mask_host && row_mask_host[i]) continue;
            const uint8_t fx = flags_host[4 * i], fz = flags_host[4 * i + 2];
            ended += fx != 0 && fz != 0;
            reached += fx != 0 && fz == 1;
        }
        const int a = cur.world_arena[w];
        if (ended && a >= 0 && a < T) {
            cur.pending[a] += ended;
            cur.pending[T + a] += reached;
        }
    }
    std::vector<int> drawn(cfg->num_worlds, -1);
    host_respawn_worlds(cfg, params,
                        [&](const LayoutConsts &c, int w) {
                            drawn[w] = weighted_arena(c, cur.cdf, T);
                            return arena_cells_draw(t, drawn[w]);
                        },
                        pose_host, goal_host, acc_host, meta_host, flags_host, live_host, status_host);
    for (int w = 0; w < cfg->num_worlds; ++w)
        if (drawn[w] >= 0 && status_host[w] == 0) cur.world_arena[w] = drawn[w];
    return RLCA_OK;
}

static int check_update(const rlca_arena_curriculum *cur, float decay, float uniform, const char *who)
{
    int rc = check_curriculum(cur, who);
    if (rc) return rc;
    if (!(decay >= 0.0f && decay < 1.0f)) return rlca_set_err(RLCA_ERR_INVALID, "%s: decay must be in [0, 1)", who);
    if (!(uniform >= 0.0f && uniform <= 1.0f))
        return rlca_set_err(RLCA_ERR_INVALID, "%s: uniform must be in [0, 1]", who);
    return RLCA_OK;
}

extern "C" int rlca_arena_curriculum_update(const rlca_arena_curriculum *curriculum, float decay, float uniform,
                                            void *stream)
{
    int rc = check_update(curriculum, decay, uniform, "rlca_arena_curriculum_update");
    if (rc) return rc;
    rlca_arena_curriculum_update_kernel<<<1, CURRICULUM_THREADS, 0, (cudaStream_t)stream>>>(
        curriculum->num_arenas, decay, uniform, curriculum->E, curriculum->S, curriculum->pending,
        reinterpret_cast<unsigned long long *>(curriculum->cdf));
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_arena_curriculum_update_host(const rlca_arena_curriculum *curriculum_host, float decay,
                                                 float uniform)
{
    int rc = check_update(curriculum_host, decay, uniform, "rlca_arena_curriculum_update_host");
    if (rc) return rc;
    const rlca_arena_curriculum &c = *curriculum_host;
    const int T = c.num_arenas;
    uint64_t total = 0;
    for (int a = 0; a < T; ++a) {
        const uint32_t w = curriculum_fold(c.E[a], c.S[a], c.pending[a], c.pending[T + a], decay, uniform);
        c.pending[a] = 0;
        c.pending[T + a] = 0;
        c.cdf[a] = total;
        total += w;
    }
    c.cdf[T] = total;
    return RLCA_OK;
}
