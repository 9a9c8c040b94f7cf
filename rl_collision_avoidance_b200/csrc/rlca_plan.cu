// rlca_plan.cu — a global planner on the device (sm_90a), C ABI in include/rlca.h, DESIGN.md §9w.
//
// Graph: the traversable cells of the map (planner.py: arenas.placeable_mask, one label per 4-connected component and
// its bounding rectangle), 8-neighbour moves of cost 70 (orthogonal) and 99 (diagonal, 99 / 70 ~ sqrt 2), a diagonal
// move only where both orthogonal neighbours are traversable.
//
// rlca_plan_fields: per row, the goal entry cell (the goal's cell if traversable, else the traversable cell of its 5 x 5
// neighbourhood whose centre is nearest the goal, ties in row-major order).  Rows whose entry changed are listed by a
// thread-per-row pass; a persistent grid of CTAs then computes each listed row's geodesic field D over its component's
// rectangle in shared memory by relaxation sweeps until a block-wide vote finds no change, and stores it in the row's
// slot.  The integer fixed point is unique, so the host twin (raster sweeps over the same relax_cell) gives the same
// bits.  A launch in which no entry changed lists nothing and every CTA of the field launch exits at once.
//
// rlca_plan_waypoints: one warp per row, from the pose and goal of the state the tick wrote.  Goal visible from the
// robot (segment_clear): status 0 and gs_out = gs_in.  Otherwise the chain of CHAIN_STEPS steepest-descent steps from
// the robot's entry cell, two chain cells per lane; the farthest visible chain cell's centre (the first chain cell when
// none is) becomes the local goal, status 1.  No plan for the goal or no entry cell for the robot: status 2, gs_in.
//
// rlca_plan_track / rlca_plan_reduce: the geodesic length L = D(start entry) res / 70 of every episode, read at the
// tracker's episode boundaries as rlca_progress_track reads them, and its per-world float64 sums.
//
// Every function the kernels call is __host__ __device__ and the file is built without contraction on either side, so
// the host twins equal the kernels bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define PLAN_INF 0xFFFFFFFFu      // not in the component (outside the field: no path)
#define PLAN_UNSET 0xFFFFFFFEu    // in the component, not reached yet (inside the field computation only)
#define COST_ORTHO 70u
#define COST_DIAG 99u
// Steps of the descent chain: one per lane and a second one per lane in a warp, 64 cells (12.8 m straight at 0.2 m),
// farther than a waypoint needs to be from the robot: the local goal is always the farthest visible cell of it.
#define CHAIN_STEPS 64
#define LIST_THREADS 256
#define FIELD_THREADS 512
#define WP_THREADS 256
#define TRACK_THREADS 128
#define REDUCE_THREADS 128

struct PlanMap {
    int gw, gh, ocx, ocy, K, max_area;
    float ppm, res;
    const int32_t *label;
    const int4 *rects;
};

// ------------------------------------------------------------------------------------------------ cells
__host__ __device__ __forceinline__ int cell_label(const PlanMap &m, int cx, int cy)
{
    return (cx >= 0 && cy >= 0 && cx < m.gw && cy < m.gh) ? m.label[cy * m.gw + cx] : -1;
}

// a coordinate in cell units (x ppm) far beyond any map: no cell, no walk
__host__ __device__ __forceinline__ bool on_scale(float u) { return fabsf(u) < 1.0e6f; }

// the tick's cell rule: cell = floor(x ppm) + origin; false for a point beyond any map
__host__ __device__ __forceinline__ bool cell_of(const PlanMap &m, float x, float y, int &cx, int &cy)
{
    const float u = x * m.ppm, v = y * m.ppm;
    if (!on_scale(u) || !on_scale(v)) return false;
    cx = (int)floorf(u) + m.ocx;
    cy = (int)floorf(v) + m.ocy;
    return true;
}

// goal entry cell cy grid_w + cx of the goal point (gx, gy), -1 = none
__host__ __device__ inline int goal_entry(const PlanMap &m, float gx, float gy)
{
    int cx, cy;
    if (!cell_of(m, gx, gy, cx, cy)) return -1;
    if (cell_label(m, cx, cy) >= 0) return cy * m.gw + cx;
    const float fx = gx * m.ppm, fy = gy * m.ppm;         // cell units relative to the origin
    int best = -1;
    float bd = 0.0f;
    for (int dy = -2; dy <= 2; ++dy)
        for (int dx = -2; dx <= 2; ++dx) {
            const int x = cx + dx, y = cy + dy;
            if (cell_label(m, x, y) < 0) continue;
            const float ex = ((float)(x - m.ocx) + 0.5f) - fx, ey = ((float)(y - m.ocy) + 0.5f) - fy;
            const float d = ex * ex + ey * ey;
            if (best < 0 || d < bd) {
                best = y * m.gw + x;
                bd = d;
            }
        }
    return best;
}

// D of cell (cx, cy) in a row's field over rectangle r (x0, y0, x1, y1); PLAN_INF outside it
__host__ __device__ __forceinline__ uint32_t field_at(const uint32_t *f, int4 r, int cx, int cy)
{
    if (cx < r.x || cx > r.z || cy < r.y || cy > r.w) return PLAN_INF;
    return f[(size_t)(cy - r.y) * (r.z - r.x + 1) + (cx - r.x)];
}

__host__ __device__ __forceinline__ uint32_t via(uint32_t d, uint32_t cost) { return d < PLAN_UNSET ? d + cost : PLAN_INF; }

// The least of D(i) and D(n) + cost(n) over the allowed moves into window cell i = y w + x of a w x h window D
// (PLAN_INF = not in the component, PLAN_UNSET = not reached yet)
__host__ __device__ __forceinline__ uint32_t relax_cell(const uint32_t *D, int w, int h, int x, int y)
{
    const int i = y * w + x;
    const bool e = x + 1 < w, wv = x > 0, n = y + 1 < h, s = y > 0;
    const uint32_t dE = e ? D[i + 1] : PLAN_INF, dW = wv ? D[i - 1] : PLAN_INF;
    const uint32_t dN = n ? D[i + w] : PLAN_INF, dS = s ? D[i - w] : PLAN_INF;
    uint32_t b = D[i];
    b = min(b, via(dE, COST_ORTHO));
    b = min(b, via(dW, COST_ORTHO));
    b = min(b, via(dN, COST_ORTHO));
    b = min(b, via(dS, COST_ORTHO));
    if (dE != PLAN_INF && dN != PLAN_INF) b = min(b, via(D[i + w + 1], COST_DIAG));
    if (dW != PLAN_INF && dN != PLAN_INF) b = min(b, via(D[i + w - 1], COST_DIAG));
    if (dW != PLAN_INF && dS != PLAN_INF) b = min(b, via(D[i - w - 1], COST_DIAG));
    if (dE != PLAN_INF && dS != PLAN_INF) b = min(b, via(D[i - w + 1], COST_DIAG));
    return b;
}

// the initial value of window cell (x, y) of a field with entry e of component comp over rectangle r
__host__ __device__ __forceinline__ uint32_t field_init(const PlanMap &m, int4 r, int e, int comp, int x, int y)
{
    const int cx = r.x + x, cy = r.y + y;
    return cy * m.gw + cx == e ? 0u : m.label[cy * m.gw + cx] == comp ? PLAN_UNSET : PLAN_INF;
}

// The robot's entry cell in component comp: its own cell when it lies in comp, else the cell of least D in its 5 x 5
// neighbourhood (ties in row-major order); false when there is none.
__host__ __device__ inline bool robot_entry(const PlanMap &m, const uint32_t *f, int4 r, int comp, int cx, int cy,
                                            int &ex, int &ey)
{
    if (cell_label(m, cx, cy) == comp) {
        ex = cx;
        ey = cy;
        return true;
    }
    uint32_t best = PLAN_INF;
    for (int dy = -2; dy <= 2; ++dy)
        for (int dx = -2; dx <= 2; ++dx) {
            const uint32_t d = field_at(f, r, cx + dx, cy + dy);
            if (d < best) {
                best = d;
                ex = cx + dx;
                ey = cy + dy;
            }
        }
    return best != PLAN_INF;
}

// One steepest-descent step from (cx, cy): the allowed neighbour of least D, ties in the order E, N, W, S, NE, NW, SW,
// SE; false when no neighbour is in the component.
__host__ __device__ inline bool descend(const uint32_t *f, int4 r, int &cx, int &cy)
{
    const int ox[4] = {1, 0, -1, 0}, oy[4] = {0, 1, 0, -1};
    uint32_t d4[4];
    uint32_t best = PLAN_INF;
    int bx = 0, by = 0;
    for (int k = 0; k < 4; ++k) {
        d4[k] = field_at(f, r, cx + ox[k], cy + oy[k]);
        if (d4[k] < best) {
            best = d4[k];
            bx = ox[k];
            by = oy[k];
        }
    }
    // NE (E, N), NW (W, N), SW (W, S), SE (E, S)
    const int dxs[4] = {1, -1, -1, 1}, dys[4] = {1, 1, -1, -1}, ka[4] = {0, 2, 2, 0}, kb[4] = {1, 1, 3, 3};
    for (int k = 0; k < 4; ++k) {
        if (d4[ka[k]] == PLAN_INF || d4[kb[k]] == PLAN_INF) continue;
        const uint32_t d = field_at(f, r, cx + dxs[k], cy + dys[k]);
        if (d < best) {
            best = d;
            bx = dxs[k];
            by = dys[k];
        }
    }
    if (best == PLAN_INF) return false;
    cx += bx;
    cy += by;
    return true;
}

__host__ __device__ __forceinline__ bool near_cell(int i, int j, int ci, int cj)
{
    return abs(i - ci) <= 1 && abs(j - cj) <= 1;
}

// Is every cell the closed segment (ax, ay) -> (bx, by) meets traversable, but for the cells within chessboard distance
// 1 of either end point's cell?  Points in cell units relative to the map origin (x ppm): a float32 supercover walk,
// column by column, of the segment's y range within each column.
__host__ __device__ inline bool segment_clear(const PlanMap &m, float ax, float ay, float bx, float by)
{
    if (!on_scale(ax) || !on_scale(ay) || !on_scale(bx) || !on_scale(by)) return false;
    if (ax > bx) {
        float t = ax; ax = bx; bx = t;
        t = ay; ay = by; by = t;
    }
    const int i0 = (int)floorf(ax), i1 = (int)floorf(bx), ja = (int)floorf(ay), jb = (int)floorf(by);
    const float slope = i1 > i0 ? (by - ay) / (bx - ax) : 0.0f;
    for (int i = i0; i <= i1; ++i) {
        float yl = ay, yr = by;
        if (i > i0) yl = ay + ((float)i - ax) * slope;
        if (i < i1) yr = ay + ((float)(i + 1) - ax) * slope;
        const int j0 = (int)floorf(fminf(yl, yr)), j1 = (int)floorf(fmaxf(yl, yr));
        for (int j = j0; j <= j1; ++j) {
            if (near_cell(i, j, i0, ja) || near_cell(i, j, i1, jb)) continue;
            if (cell_label(m, i + m.ocx, j + m.ocy) < 0) return false;
        }
    }
    return true;
}

// the centre of map cell (cx, cy) in cell units relative to the origin
__host__ __device__ __forceinline__ float centre_u(int c, int oc) { return (float)(c - oc) + 0.5f; }

// L of a start point: D(start entry) res / 70 m, -1 = no path (no plan for the goal, or no entry cell)
__host__ __device__ inline float geo_length(const PlanMap &m, int e, const uint32_t *f, int4 r, float x, float y)
{
    if (e < 0) return -1.0f;
    int cx, cy, ex, ey;
    if (!cell_of(m, x, y, cx, cy)) return -1.0f;
    if (!robot_entry(m, f, r, m.label[e], cx, cy, ex, ey)) return -1.0f;
    const uint32_t d = field_at(f, r, ex, ey);
    return (float)((double)d * (double)m.res / 70.0);
}

// ------------------------------------------------------------------------------------------------ fields
__global__ void __launch_bounds__(LIST_THREADS) rlca_plan_list_kernel(PlanMap m, int n, const float4 *__restrict__ goal,
                                                                      int32_t *__restrict__ entry, int4 *__restrict__ rect,
                                                                      int32_t *__restrict__ list)
{
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n) return;
    const float4 g = goal[a];
    const int e = goal_entry(m, g.x, g.y);
    if (e == entry[a]) return;
    entry[a] = e;
    if (e < 0) return;
    rect[a] = m.rects[m.label[e]];
    list[1 + atomicAdd(list, 1)] = a;
}

__global__ void __launch_bounds__(FIELD_THREADS) rlca_plan_field_kernel(PlanMap m, const int32_t *__restrict__ list,
                                                                        const int32_t *__restrict__ entry,
                                                                        const int4 *__restrict__ rect,
                                                                        uint32_t *__restrict__ field)
{
    extern __shared__ uint32_t D[];
    const int count = list[0];
    for (int k = blockIdx.x; k < count; k += gridDim.x) {
        const int row = list[1 + k];
        const int e = entry[row];
        const int4 r = rect[row];
        const int w = r.z - r.x + 1, h = r.w - r.y + 1, A = w * h, comp = m.label[e];
        for (int i = threadIdx.x; i < A; i += blockDim.x) D[i] = field_init(m, r, e, comp, i % w, i / w);
        __syncthreads();
        // sweeps alternate their order, so that a front travels both ways along the window's rows within a sweep.
        // A cell's owner is its only writer; a neighbour read mid-sweep is an old or a new value, both upper bounds.
        int sweep = 0, changed;
        do {
            changed = 0;
            for (int t = threadIdx.x; t < A; t += blockDim.x) {
                const int i = (sweep & 1) ? A - 1 - t : t;
                const uint32_t d = D[i];
                if (d == PLAN_INF) continue;
                const uint32_t b = relax_cell(D, w, h, i % w, i / w);
                if (b < d) {
                    D[i] = b;
                    changed = 1;
                }
            }
            ++sweep;
        } while (__syncthreads_or(changed));
        uint32_t *out = field + (size_t)row * m.max_area;
        for (int i = threadIdx.x; i < A; i += blockDim.x) out[i] = D[i];
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ waypoints
// One row's plan; lane `lane` of 32 tests chain cells lane and lane + 32 (the host twin passes lane -1 and tests all).
// Returns the status; gs and the waypoint's cell (wx, wy) are written for status 1 only.
struct RowIn {
    float4 pose, goal;
    int e;
    int4 r;
    const uint32_t *f;
};

__host__ __device__ inline bool chain_visible(const PlanMap &m, const RowIn &q, int cx, int cy)
{
    return segment_clear(m, q.pose.x * m.ppm, q.pose.y * m.ppm, centre_u(cx, m.ocx), centre_u(cy, m.ocy));
}

__device__ __forceinline__ int warp_row(const PlanMap &m, const RowIn &q, int lane, float4 &gs, int &wx, int &wy)
{
    int cx, cy, ex, ey;
    if (q.e < 0 || !cell_of(m, q.pose.x, q.pose.y, cx, cy)) return 2;
    if (segment_clear(m, q.pose.x * m.ppm, q.pose.y * m.ppm, q.goal.x * m.ppm, q.goal.y * m.ppm)) return 0;
    if (!robot_entry(m, q.f, q.r, m.label[q.e], cx, cy, ex, ey)) return 2;
    // the chain, every lane walking it and keeping cells lane and lane + 32
    int len = 0, c0x = ex, c0y = ey, c1x = ex, c1y = ey;
    if (field_at(q.f, q.r, ex, ey) == 0) {
        len = 1;
    } else {
        int x = ex, y = ey;
        while (len < CHAIN_STEPS && field_at(q.f, q.r, x, y) != 0 && descend(q.f, q.r, x, y)) {
            if (len == lane) { c0x = x; c0y = y; }
            if (len == lane + 32) { c1x = x; c1y = y; }
            ++len;
        }
        if (len == 0) len = 1;                  // no step (cannot happen on an exact field): the entry cell
    }
    const bool v0 = lane < len && chain_visible(m, q, c0x, c0y);
    const bool v1 = lane + 32 < len && chain_visible(m, q, c1x, c1y);
    const unsigned b0 = __ballot_sync(0xFFFFFFFFu, v0), b1 = __ballot_sync(0xFFFFFFFFu, v1);
    const int best = b1 ? 63 - __clz(b1) : b0 ? 31 - __clz(b0) : 0;
    const int src = best & 31;
    wx = __shfl_sync(0xFFFFFFFFu, best >= 32 ? c1x : c0x, src);
    wy = __shfl_sync(0xFFFFFFFFu, best >= 32 ? c1y : c0y, src);
    float s, c;
    dev_sincosf(q.pose.z, s, c);
    gs = goal_speed(q.pose, make_float4(centre_u(wx, m.ocx) * m.res, centre_u(wy, m.ocy) * m.res, q.goal.z, q.goal.w),
                    s, c);
    return 1;
}

// the host twin of warp_row: the same functions, the chain in one array
static int host_row(const PlanMap &m, const RowIn &q, float4 &gs, int &wx, int &wy)
{
    int cx, cy, ex, ey;
    if (q.e < 0 || !cell_of(m, q.pose.x, q.pose.y, cx, cy)) return 2;
    if (segment_clear(m, q.pose.x * m.ppm, q.pose.y * m.ppm, q.goal.x * m.ppm, q.goal.y * m.ppm)) return 0;
    if (!robot_entry(m, q.f, q.r, m.label[q.e], cx, cy, ex, ey)) return 2;
    int chx[CHAIN_STEPS], chy[CHAIN_STEPS], len = 0;
    if (field_at(q.f, q.r, ex, ey) != 0) {
        int x = ex, y = ey;
        while (len < CHAIN_STEPS && field_at(q.f, q.r, x, y) != 0 && descend(q.f, q.r, x, y)) {
            chx[len] = x;
            chy[len] = y;
            ++len;
        }
    }
    if (len == 0) {
        chx[0] = ex;
        chy[0] = ey;
        len = 1;
    }
    int best = 0;
    for (int k = 0; k < len; ++k)
        if (chain_visible(m, q, chx[k], chy[k])) best = k;
    wx = chx[best];
    wy = chy[best];
    float s, c;
    dev_sincosf(q.pose.z, s, c);
    gs = goal_speed(q.pose, make_float4(centre_u(wx, m.ocx) * m.res, centre_u(wy, m.ocy) * m.res, q.goal.z, q.goal.w),
                    s, c);
    return 1;
}

// ------------------------------------------------------------------------------------------------ shaped reward
// The geodesic progress potential phi = pose.w + psi of a row after a tick: psi = 0 for status 0 (goal visible) and 2
// (no plan), and for status 1 the distance to the waypoint w plus the waypoint cell's remaining geodesic length, less
// the straight-line distance pose.w the tick stored: psi = (|p - w| + D(c_w) res / 70) - pose.w.
__host__ __device__ inline float psi_excess(const PlanMap &m, const RowIn &q, int st, int wx, int wy)
{
    if (st != 1) return 0.0f;
    const float dx = centre_u(wx, m.ocx) * m.res - q.pose.x, dy = centre_u(wy, m.ocy) * m.res - q.pose.y;
    const float L = (float)((double)field_at(q.f, q.r, wx, wy) * (double)m.res / 70.0);
    return (sqrtf(fmaf(dx, dx, dy * dy)) + L) - q.pose.w;
}

// The per-row buffers and outputs of the shaping launch; flags NULL at a run's start (reward and eplog unused)
struct ShapeIo {
    float gain;
    const uchar4 *flags;
    float *reward, *eplog, *psi_prev, *psi_start;
};

// Row a's shaping with its new psi: a non-terminal tick (flags.x == 0) adds gain (psi_prev - psi) to the tick's reward;
// a tick that wrote the row's eplog (flags.x and flags.z) adds gain (psi_start - psi_prev) to its return, the sum of
// the episode's shaping terms; every other reward stays the tick's.  Then psi_prev = psi, and psi_start = psi at an
// episode start (flags.w, or every row at a run's start).
__host__ __device__ inline void shape_row(const ShapeIo &sh, int a, float psi)
{
    bool start = true;
    if (sh.flags) {
        const uchar4 fl = sh.flags[a];
        const float pp = sh.psi_prev[a];
        if (fl.x == 0) {
            sh.reward[a] = sh.reward[a] + sh.gain * (pp - psi);
        } else if (fl.z != 0 && sh.eplog) {
            float &ret = sh.eplog[(size_t)a * 8 + 2];
            ret = ret + sh.gain * (sh.psi_start[a] - pp);
        }
        start = fl.w != 0;
    }
    sh.psi_prev[a] = psi;
    if (start) sh.psi_start[a] = psi;
}

__global__ void __launch_bounds__(WP_THREADS) rlca_plan_waypoints_kernel(
    PlanMap m, int n, const float4 *__restrict__ pose, const float4 *__restrict__ goal, const int32_t *__restrict__ entry,
    const int4 *__restrict__ rect, const uint32_t *__restrict__ field, const float4 *__restrict__ gs_in,
    float4 *__restrict__ gs_out, uint8_t *__restrict__ status, int32_t *__restrict__ status_count)
{
    const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= n) return;                                 // warp-uniform
    RowIn q;
    q.pose = pose[a];
    const float4 g = goal[a], in = gs_in[a];            // a waypoint replaces the local goal, never the speed
    q.goal = make_float4(g.x, g.y, in.z, in.w);
    q.e = entry[a];
    q.r = q.e >= 0 ? rect[a] : make_int4(0, 0, -1, -1);
    q.f = field + (size_t)a * m.max_area;
    float4 gs = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    int wx, wy;
    const int st = warp_row(m, q, lane, gs, wx, wy);
    if (lane == 0) {
        gs_out[a] = st == 1 ? gs : in;
        status[a] = (uint8_t)st;
        status_count[3 * a + st] += 1;
    }
}

// rlca_plan_waypoints_kernel's rows and, on lane 0, the row's psi and shaping.  Lane 0 reads the row's gs_in before it
// writes gs_out, so gs_in and gs_out may be one buffer: neither is __restrict__.  (The waypoint kernel keeps its own
// copy of these few lines: sharing them through a template body reorders two of its instructions.)
__global__ void __launch_bounds__(WP_THREADS) rlca_plan_shape_kernel(
    PlanMap m, int n, ShapeIo sh, const float4 *__restrict__ pose, const float4 *__restrict__ goal,
    const int32_t *__restrict__ entry, const int4 *__restrict__ rect, const uint32_t *__restrict__ field,
    const float4 *gs_in, float4 *gs_out, uint8_t *__restrict__ status, int32_t *__restrict__ status_count)
{
    const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= n) return;                                 // warp-uniform
    RowIn q;
    q.pose = pose[a];
    q.goal = goal[a];
    q.e = entry[a];
    q.r = q.e >= 0 ? rect[a] : make_int4(0, 0, -1, -1);
    q.f = field + (size_t)a * m.max_area;
    float4 gs = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    int wx, wy;                                         // written for status 1, the only status psi_excess reads
    const int st = warp_row(m, q, lane, gs, wx, wy);
    if (lane == 0) {
        float4 out = gs_in[a];                          // a waypoint replaces the local goal, never the speed
        if (st == 1) { out.x = gs.x; out.y = gs.y; }
        gs_out[a] = out;
        status[a] = (uint8_t)st;
        status_count[3 * a + st] += 1;
        shape_row(sh, a, psi_excess(m, q, st, wx, wy));
    }
}

// the host twin of both kernels over every row (sh NULL: rlca_plan_waypoints_kernel)
static void host_rows(const PlanMap &m, int n, const rlca_plan_state *ps, const rlca_env_state *state,
                      const float *gs_in_host, float *gs_out_host, const ShapeIo *sh)
{
    const float4 *pose = reinterpret_cast<const float4 *>(state->pose_dev);
    const float4 *goal = reinterpret_cast<const float4 *>(state->goal_dev);
    const int4 *rect = reinterpret_cast<const int4 *>(ps->rect);
    const float4 *gs_in = reinterpret_cast<const float4 *>(gs_in_host);
    float4 *gs_out = reinterpret_cast<float4 *>(gs_out_host);
    for (int a = 0; a < n; ++a) {
        RowIn q;
        q.pose = pose[a];
        q.goal = goal[a];
        q.e = ps->entry[a];
        q.r = q.e >= 0 ? rect[a] : make_int4(0, 0, -1, -1);
        q.f = ps->field + (size_t)a * m.max_area;
        float4 gs = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        int wx = 0, wy = 0;
        const int st = host_row(m, q, gs, wx, wy);
        float4 out = gs_in[a];
        if (st == 1) { out.x = gs.x; out.y = gs.y; }
        gs_out[a] = out;
        ps->status[a] = (uint8_t)st;
        ps->status_count[3 * a + st] += 1;
        if (sh) shape_row(*sh, a, psi_excess(m, q, st, wx, wy));
    }
}

// ------------------------------------------------------------------------------------------------ geodesic tracker
// Row a after a tick (flags != NULL) or at a run's start (flags == NULL: every row starts an episode).  A tracked
// episode that ends writes its L into the tracker's next slot; then an episode start (a re-spawn, flags.w) computes the
// new L from the episode's init pose (acc.zw) and the field of the goal it now has.
__host__ __device__ inline void track_row(const PlanMap &m, int a, int episodes, const int4 *meta_in, const float4 *acc,
                                          const uchar4 *flags, const int32_t *closed, const int32_t *count,
                                          const int32_t *entry, const int4 *rect, const uint32_t *field, float *length,
                                          float *records)
{
    bool start = true;
    if (flags) {
        const uchar4 fl = flags[a];
        const bool tracked = closed[a] != meta_in[a].y;
        const int c = count[a];
        if (tracked && fl.z != 0 && c < episodes) records[(size_t)a * episodes + c] = length[a];
        start = fl.w != 0;
    }
    if (start) {
        const int e = entry[a];
        const int4 r = e >= 0 ? rect[a] : make_int4(0, 0, -1, -1);
        const float4 p = acc[a];
        length[a] = geo_length(m, e, field + (size_t)a * m.max_area, r, p.z, p.w);
    }
}

__global__ void __launch_bounds__(TRACK_THREADS) rlca_plan_track_kernel(
    PlanMap m, int n, int episodes, const int4 *__restrict__ meta_in, const float4 *__restrict__ acc,
    const uchar4 *__restrict__ flags, const int32_t *__restrict__ closed, const int32_t *__restrict__ count,
    const int32_t *__restrict__ entry, const int4 *__restrict__ rect, const uint32_t *__restrict__ field,
    float *__restrict__ length, float *__restrict__ records)
{
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n) return;
    track_row(m, a, episodes, meta_in, acc, flags, closed, count, entry, rect, field, length, records);
}

// ------------------------------------------------------------------------------------------------ reduction
// Partials of world w, layout RLCA_PLAN_* of include/rlca.h; with a mask only the agents whose (mask != 0) equals want
__host__ __device__ inline void plan_reduce_world(int R, int episodes, double goal_radius, const float *geo,
                                                  const float4 *erec, const int32_t *count, int w, const uint8_t *mask,
                                                  bool want, double *out)
{
    double s[RLCA_PLAN_NPARTIALS];
    for (int k = 0; k < RLCA_PLAN_NPARTIALS; ++k) s[k] = 0.0;
    for (int r = 0; r < R; ++r) {
        const int a = w * R + r;
        if (mask && (mask[a] != 0) != want) continue;
        const int c = count[a];
        const int nrec = c < episodes ? c : episodes;
        for (int i = 0; i < nrec; ++i) {
            const size_t k = (size_t)a * episodes + i;
            const float L = geo[k];
            if (!(L >= 0.0f)) {
                s[RLCA_PLAN_NO_PATH] = d_add(s[RLCA_PLAN_NO_PATH], 1.0);
                continue;
            }
            if ((int)erec[k].x != 1) continue;
            const double Ld = (double)L, Lr = d_add(Ld, -goal_radius);
            const double x = d_add((double)erec[k].z, -(Lr > 0.0 ? Lr : 0.0));
            s[RLCA_PLAN_REACHED] = d_add(s[RLCA_PLAN_REACHED], 1.0);
            s[RLCA_PLAN_SUM_LENGTH] = d_add(s[RLCA_PLAN_SUM_LENGTH], Ld);
            s[RLCA_PLAN_SUM_EXTRA] = d_add(s[RLCA_PLAN_SUM_EXTRA], x);
            s[RLCA_PLAN_SUM_EXTRA_SQ] = d_add(s[RLCA_PLAN_SUM_EXTRA_SQ], d_mul(x, x));
        }
    }
    for (int k = 0; k < RLCA_PLAN_NPARTIALS; ++k) out[k] = s[k];
}

__global__ void __launch_bounds__(REDUCE_THREADS) rlca_plan_reduce_kernel(int R, int episodes, double goal_radius,
                                                                          const float *geo, const float4 *erec,
                                                                          const int32_t *count, const uint8_t *mask,
                                                                          int world_begin, int world_count,
                                                                          double *partials)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, rows = mask ? 2 : 1;
    if (i >= rows * world_count) return;
    plan_reduce_world(R, episodes, goal_radius, geo, erec, count, world_begin + i / rows, mask, i % rows,
                      partials + (size_t)i * RLCA_PLAN_NPARTIALS);
}

// ------------------------------------------------------------------------------------------------ entries
static int plan_args(const char *who, const rlca_env_config *cfg, const rlca_plan_tables *t, const rlca_plan_state *ps,
                     PlanMap &m)
{
    if (!cfg || !t || !ps) return rlca_set_err(RLCA_ERR_INVALID, "%s: cfg, tables or plan state is NULL", who);
    if (int rc = rlca_check_robots(cfg, who)) return rc;
    if (cfg->grid_w < 1 || cfg->grid_h < 1 || !(cfg->ppm > 0.0f) || !(cfg->resolution > 0.0f))
        return rlca_set_err(RLCA_ERR_INVALID, "%s: the config has no map", who);
    if (t->num_components < 1 || t->max_area < 1 || t->max_area > RLCA_PLAN_MAX_CELLS || !t->label || !t->rects)
        return rlca_set_err(RLCA_ERR_INVALID,
                            "%s: tables need num_components >= 1, max_area in 1..RLCA_PLAN_MAX_CELLS, label and rects",
                            who);
    m.gw = cfg->grid_w;
    m.gh = cfg->grid_h;
    m.ocx = cfg->origin_cx;
    m.ocy = cfg->origin_cy;
    m.K = t->num_components;
    m.max_area = t->max_area;
    m.ppm = cfg->ppm;
    m.res = cfg->resolution;
    m.label = t->label;
    m.rects = reinterpret_cast<const int4 *>(t->rects);
    return RLCA_OK;
}

extern "C" int rlca_plan_tables_check(const rlca_env_config *cfg, const rlca_plan_tables *t)
{
    if (!cfg || !t) return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_tables_check: cfg or tables is NULL");
    if (cfg->grid_w < 1 || cfg->grid_h < 1) return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_tables_check: no map");
    if (t->num_components < 1 || !t->label || !t->rects)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_tables_check: no component, or a NULL label or rects");
    if (t->max_area < 1 || t->max_area > RLCA_PLAN_MAX_CELLS)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_tables_check: max_area outside 1..RLCA_PLAN_MAX_CELLS");
    const int K = t->num_components;
    for (int k = 0; k < K; ++k) {
        const int *r = t->rects + 4 * k;
        if (r[0] < 0 || r[1] < 0 || r[2] < r[0] || r[3] < r[1] || r[2] >= cfg->grid_w || r[3] >= cfg->grid_h)
            return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_tables_check: a rectangle is empty or leaves the grid");
        if ((int64_t)(r[2] - r[0] + 1) * (r[3] - r[1] + 1) > t->max_area)
            return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_tables_check: a rectangle holds more than max_area cells");
    }
    for (int y = 0; y < cfg->grid_h; ++y)
        for (int x = 0; x < cfg->grid_w; ++x) {
            const int l = t->label[y * cfg->grid_w + x];
            if (l < -1 || l >= K) return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_tables_check: a label is out of range");
            if (l >= 0) {
                const int *r = t->rects + 4 * l;
                if (x < r[0] || x > r[2] || y < r[1] || y > r[3])
                    return rlca_set_err(RLCA_ERR_INVALID,
                                        "rlca_plan_tables_check: a cell lies outside its component's rectangle");
            }
        }
    return RLCA_OK;
}

extern "C" int rlca_plan_fields(const rlca_env_config *cfg, const rlca_plan_tables *tables, const rlca_plan_state *ps,
                                const rlca_env_state *state, void *stream)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_fields", cfg, tables, ps, m);
    if (rc) return rc;
    if (!state || !state->goal_dev || !ps->entry || !ps->rect || !ps->field || !ps->list)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_fields: a buffer is NULL");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const size_t smem = (size_t)m.max_area * sizeof(uint32_t);
    cudaStream_t s = (cudaStream_t)stream;
    RLCA_CUDA_TRY(cudaFuncSetAttribute(rlca_plan_field_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, sms = 0, per_sm = 0;
    RLCA_CUDA_TRY(cudaGetDevice(&dev));
    RLCA_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    RLCA_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rlca_plan_field_kernel, FIELD_THREADS, smem));
    if (per_sm < 1) return rlca_set_err(RLCA_ERR_UNSUPPORTED, "rlca_plan_fields: a field does not fit one CTA");
    const int grid = n < sms * per_sm ? n : sms * per_sm;
    RLCA_CUDA_TRY(cudaMemsetAsync(ps->list, 0, sizeof(int32_t), s));
    rlca_plan_list_kernel<<<(n + LIST_THREADS - 1) / LIST_THREADS, LIST_THREADS, 0, s>>>(
        m, n, reinterpret_cast<const float4 *>(state->goal_dev), ps->entry, reinterpret_cast<int4 *>(ps->rect), ps->list);
    RLCA_CUDA_TRY(cudaGetLastError());
    rlca_plan_field_kernel<<<grid, FIELD_THREADS, smem, s>>>(m, ps->list, ps->entry,
                                                             reinterpret_cast<const int4 *>(ps->rect), ps->field);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_plan_fields_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                                     const rlca_plan_state *ps_host, const rlca_env_state *state_host)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_fields_host", cfg, tables_host, ps_host, m);
    if (rc) return rc;
    if ((rc = rlca_plan_tables_check(cfg, tables_host))) return rc;
    if (!state_host || !state_host->goal_dev || !ps_host->entry || !ps_host->rect || !ps_host->field || !ps_host->list)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_fields_host: a buffer is NULL");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const float4 *goal = reinterpret_cast<const float4 *>(state_host->goal_dev);
    int4 *rect = reinterpret_cast<int4 *>(ps_host->rect);
    uint32_t *D = (uint32_t *)malloc((size_t)m.max_area * sizeof(uint32_t));
    if (!D) return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_fields_host: out of host memory");
    int32_t *list = ps_host->list;
    list[0] = 0;
    for (int a = 0; a < n; ++a) {
        const int e = goal_entry(m, goal[a].x, goal[a].y);
        if (e == ps_host->entry[a]) continue;
        ps_host->entry[a] = e;
        if (e < 0) continue;
        const int4 r = m.rects[m.label[e]];
        rect[a] = r;
        list[1 + list[0]++] = a;
        const int w = r.z - r.x + 1, h = r.w - r.y + 1, A = w * h, comp = m.label[e];
        for (int i = 0; i < A; ++i) D[i] = field_init(m, r, e, comp, i % w, i / w);
        // raster sweeps, forward then backward, until one changes nothing
        for (int sweep = 0, changed = 1; changed; ++sweep) {
            changed = 0;
            for (int t = 0; t < A; ++t) {
                const int i = (sweep & 1) ? A - 1 - t : t;
                if (D[i] == PLAN_INF) continue;
                const uint32_t b = relax_cell(D, w, h, i % w, i / w);
                if (b < D[i]) {
                    D[i] = b;
                    changed = 1;
                }
            }
        }
        uint32_t *out = ps_host->field + (size_t)a * m.max_area;
        for (int i = 0; i < A; ++i) out[i] = D[i];
    }
    free(D);
    return RLCA_OK;
}

extern "C" int rlca_plan_waypoints(const rlca_env_config *cfg, const rlca_plan_tables *tables,
                                   const rlca_plan_state *ps, const rlca_env_state *state, const float *gs_in_dev,
                                   float *gs_out_dev, void *stream)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_waypoints", cfg, tables, ps, m);
    if (rc) return rc;
    if (!state || !state->pose_dev || !state->goal_dev || !gs_in_dev || !gs_out_dev || !ps->entry || !ps->rect ||
        !ps->field || !ps->status || !ps->status_count)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_waypoints: a buffer is NULL");
    if (gs_in_dev == gs_out_dev) return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_waypoints: gs_in and gs_out alias");
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const int rows_per_cta = WP_THREADS / 32;
    rlca_plan_waypoints_kernel<<<(n + rows_per_cta - 1) / rows_per_cta, WP_THREADS, 0, (cudaStream_t)stream>>>(
        m, n, reinterpret_cast<const float4 *>(state->pose_dev), reinterpret_cast<const float4 *>(state->goal_dev),
        ps->entry, reinterpret_cast<const int4 *>(ps->rect), ps->field, reinterpret_cast<const float4 *>(gs_in_dev),
        reinterpret_cast<float4 *>(gs_out_dev), ps->status, ps->status_count);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_plan_waypoints_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                                        const rlca_plan_state *ps_host, const rlca_env_state *state_host,
                                        const float *gs_in_host, float *gs_out_host)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_waypoints_host", cfg, tables_host, ps_host, m);
    if (rc) return rc;
    if ((rc = rlca_plan_tables_check(cfg, tables_host))) return rc;
    if (!state_host || !state_host->pose_dev || !state_host->goal_dev || !gs_in_host || !gs_out_host ||
        !ps_host->entry || !ps_host->rect || !ps_host->field || !ps_host->status || !ps_host->status_count)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_waypoints_host: a buffer is NULL");
    if (gs_in_host == gs_out_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_waypoints_host: gs_in and gs_out alias");
    host_rows(m, cfg->robots_per_world * cfg->num_worlds, ps_host, state_host, gs_in_host, gs_out_host, nullptr);
    return RLCA_OK;
}

static int shape_args(const char *who, const rlca_plan_state *ps, const float *psi_prev, const float *psi_start,
                      const rlca_env_state *state, const uint8_t *flags, const float *reward, const float *gs_in,
                      const float *gs_out)
{
    if (!state || !state->pose_dev || !state->goal_dev || !gs_in || !gs_out || !ps->entry || !ps->rect ||
        !ps->field || !ps->status || !ps->status_count || !psi_prev || !psi_start)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: a buffer is NULL", who);
    if (psi_prev == psi_start) return rlca_set_err(RLCA_ERR_INVALID, "%s: psi_prev and psi_start alias", who);
    if (flags && !reward) return rlca_set_err(RLCA_ERR_INVALID, "%s: after a tick the reward is needed", who);
    return RLCA_OK;
}

extern "C" int rlca_plan_shape(const rlca_env_config *cfg, const rlca_plan_tables *tables, const rlca_plan_state *ps,
                               float *psi_prev_dev, float *psi_start_dev, const rlca_env_state *state,
                               const uint8_t *flags_dev, float *reward_dev, float *eplog_dev, const float *gs_in_dev,
                               float *gs_out_dev, void *stream)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_shape", cfg, tables, ps, m);
    if (rc) return rc;
    if ((rc = shape_args("rlca_plan_shape", ps, psi_prev_dev, psi_start_dev, state, flags_dev, reward_dev, gs_in_dev,
                         gs_out_dev)))
        return rc;
    ShapeIo sh;
    sh.gain = cfg->progress_gain;
    sh.flags = reinterpret_cast<const uchar4 *>(flags_dev);
    sh.reward = reward_dev;
    sh.eplog = eplog_dev;
    sh.psi_prev = psi_prev_dev;
    sh.psi_start = psi_start_dev;
    const int n = cfg->robots_per_world * cfg->num_worlds;
    const int rows_per_cta = WP_THREADS / 32;
    rlca_plan_shape_kernel<<<(n + rows_per_cta - 1) / rows_per_cta, WP_THREADS, 0, (cudaStream_t)stream>>>(
        m, n, sh, reinterpret_cast<const float4 *>(state->pose_dev), reinterpret_cast<const float4 *>(state->goal_dev),
        ps->entry, reinterpret_cast<const int4 *>(ps->rect), ps->field, reinterpret_cast<const float4 *>(gs_in_dev),
        reinterpret_cast<float4 *>(gs_out_dev), ps->status, ps->status_count);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_plan_shape_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                                    const rlca_plan_state *ps_host, float *psi_prev_host, float *psi_start_host,
                                    const rlca_env_state *state_host, const uint8_t *flags_host, float *reward_host,
                                    float *eplog_host, const float *gs_in_host, float *gs_out_host)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_shape_host", cfg, tables_host, ps_host, m);
    if (rc) return rc;
    if ((rc = rlca_plan_tables_check(cfg, tables_host))) return rc;
    if ((rc = shape_args("rlca_plan_shape_host", ps_host, psi_prev_host, psi_start_host, state_host, flags_host,
                         reward_host, gs_in_host, gs_out_host)))
        return rc;
    ShapeIo sh;
    sh.gain = cfg->progress_gain;
    sh.flags = reinterpret_cast<const uchar4 *>(flags_host);
    sh.reward = reward_host;
    sh.eplog = eplog_host;
    sh.psi_prev = psi_prev_host;
    sh.psi_start = psi_start_host;
    host_rows(m, cfg->robots_per_world * cfg->num_worlds, ps_host, state_host, gs_in_host, gs_out_host, &sh);
    return RLCA_OK;
}

static int track_args(const char *who, const rlca_plan_state *ps, const rlca_env_state *state_in,
                      const rlca_env_state *state_out, const uint8_t *flags, const int32_t *closed,
                      const int32_t *count, int32_t episodes)
{
    if (!state_out || !state_out->acc_dev || !ps->entry || !ps->rect || !ps->field || !ps->length || !ps->records)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: a buffer is NULL", who);
    if (ps->episodes < 1 || ps->episodes != episodes)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: episodes must be >= 1 and the tracker's", who);
    if (flags && (!state_in || !state_in->meta_dev || !closed || !count))
        return rlca_set_err(RLCA_ERR_INVALID, "%s: after a tick state_in, its meta, closed and count are needed", who);
    return RLCA_OK;
}

extern "C" int rlca_plan_track(const rlca_env_config *cfg, const rlca_plan_tables *tables, const rlca_plan_state *ps,
                               const rlca_env_state *state_in, const rlca_env_state *state_out, const uint8_t *flags_dev,
                               const rlca_eval_state *ev, void *stream)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_track", cfg, tables, ps, m);
    if (rc) return rc;
    if (!ev) return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_track: eval state is NULL");
    if ((rc = track_args("rlca_plan_track", ps, state_in, state_out, flags_dev, ev->closed_dev, ev->count_dev,
                         ev->episodes)))
        return rc;
    const int n = cfg->robots_per_world * cfg->num_worlds;
    rlca_plan_track_kernel<<<(n + TRACK_THREADS - 1) / TRACK_THREADS, TRACK_THREADS, 0, (cudaStream_t)stream>>>(
        m, n, ps->episodes, flags_dev ? reinterpret_cast<const int4 *>(state_in->meta_dev) : nullptr,
        reinterpret_cast<const float4 *>(state_out->acc_dev), reinterpret_cast<const uchar4 *>(flags_dev),
        ev->closed_dev, ev->count_dev, ps->entry, reinterpret_cast<const int4 *>(ps->rect), ps->field, ps->length,
        ps->records);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_plan_track_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                                    const rlca_plan_state *ps_host, const rlca_env_state *state_in_host,
                                    const rlca_env_state *state_out_host, const uint8_t *flags_host,
                                    const int32_t *closed_host, const int32_t *count_host, int32_t episodes)
{
    PlanMap m;
    int rc = plan_args("rlca_plan_track_host", cfg, tables_host, ps_host, m);
    if (rc) return rc;
    if ((rc = rlca_plan_tables_check(cfg, tables_host))) return rc;
    if ((rc = track_args("rlca_plan_track_host", ps_host, state_in_host, state_out_host, flags_host, closed_host,
                         count_host, episodes)))
        return rc;
    const int n = cfg->robots_per_world * cfg->num_worlds;
    for (int a = 0; a < n; ++a)
        track_row(m, a, episodes, flags_host ? reinterpret_cast<const int4 *>(state_in_host->meta_dev) : nullptr,
                  reinterpret_cast<const float4 *>(state_out_host->acc_dev),
                  reinterpret_cast<const uchar4 *>(flags_host), closed_host, count_host, ps_host->entry,
                  reinterpret_cast<const int4 *>(ps_host->rect), ps_host->field, ps_host->length, ps_host->records);
    return RLCA_OK;
}

static int reduce_args(const char *who, const rlca_env_config *cfg, int32_t episodes, int32_t world_begin,
                       int32_t world_count)
{
    if (!cfg) return rlca_set_err(RLCA_ERR_INVALID, "%s: cfg is NULL", who);
    if (int rc = rlca_check_robots(cfg, who)) return rc;
    if (episodes < 1) return rlca_set_err(RLCA_ERR_INVALID, "%s: episodes must be >= 1", who);
    return rlca_check_world_range(cfg, world_begin, world_count, who);
}

static int plan_reduce_launch(const char *who, const rlca_env_config *cfg, const rlca_plan_state *ps,
                              const rlca_eval_state *ev, const uint8_t *mask_dev, int32_t world_begin,
                              int32_t world_count, double *partials_dev, void *stream)
{
    if (!ps || !ev) return rlca_set_err(RLCA_ERR_INVALID, "%s: plan state or eval state is NULL", who);
    int rc = reduce_args(who, cfg, ps->episodes, world_begin, world_count);
    if (rc) return rc;
    if (ev->episodes != ps->episodes)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: the tracker holds a different number of episodes", who);
    if (!ps->records || !ev->records_dev || !ev->count_dev || !partials_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "%s: a buffer is NULL", who);
    const int threads = (mask_dev ? 2 : 1) * world_count;
    rlca_plan_reduce_kernel<<<(threads + REDUCE_THREADS - 1) / REDUCE_THREADS, REDUCE_THREADS, 0,
                              (cudaStream_t)stream>>>(
        cfg->robots_per_world, ps->episodes, (double)cfg->goal_radius, ps->records,
        reinterpret_cast<const float4 *>(ev->records_dev), ev->count_dev, mask_dev, world_begin, world_count,
        partials_dev);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_plan_reduce(const rlca_env_config *cfg, const rlca_plan_state *ps, const rlca_eval_state *ev,
                                int32_t world_begin, int32_t world_count, double *partials_dev, void *stream)
{
    return plan_reduce_launch("rlca_plan_reduce", cfg, ps, ev, nullptr, world_begin, world_count, partials_dev, stream);
}

extern "C" int rlca_plan_reduce_split(const rlca_env_config *cfg, const rlca_plan_state *ps, const rlca_eval_state *ev,
                                      const uint8_t *mask_dev, int32_t world_begin, int32_t world_count,
                                      double *partials_dev, void *stream)
{
    if (!mask_dev) return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_reduce_split: mask is NULL");
    return plan_reduce_launch("rlca_plan_reduce_split", cfg, ps, ev, mask_dev, world_begin, world_count, partials_dev,
                              stream);
}

extern "C" int rlca_plan_reduce_host(const rlca_env_config *cfg, const float *geo_records_host,
                                     const float *eval_records_host, const int32_t *count_host,
                                     const uint8_t *mask_host, int32_t episodes, int32_t world_begin,
                                     int32_t world_count, double *partials_host)
{
    int rc = reduce_args("rlca_plan_reduce_host", cfg, episodes, world_begin, world_count);
    if (rc) return rc;
    if (!geo_records_host || !eval_records_host || !count_host || !partials_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_plan_reduce_host: a buffer is NULL");
    const int rows = mask_host ? 2 : 1;
    for (int i = 0; i < rows * world_count; ++i)
        plan_reduce_world(cfg->robots_per_world, episodes, (double)cfg->goal_radius, geo_records_host,
                          reinterpret_cast<const float4 *>(eval_records_host), count_host, world_begin + i / rows,
                          mask_host, i % rows, partials_host + (size_t)i * RLCA_PLAN_NPARTIALS);
    return RLCA_OK;
}
