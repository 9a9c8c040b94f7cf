// rlca_dynamics.cu — acceleration limits just before the tick (sm_90a), C ABI in include/rlca.h, DESIGN.md §9r.
//
// rlca_dynamics_action turns the command of a tick into the command a robot with linear and angular acceleration
// limits executes: each component moves from the velocity executed on the last call towards the command by at most
// limit * dt.  The limits are drawn per agent when it starts an episode and held until its next one.  It is a separate
// launch; the tick's kernels, its config and its outputs are untouched, and a run without limits issues none.
//
// The executed velocity and the limits are state across ticks, so this is a file of its own, as latency is.  Every
// limit is a function of (seed, global agent, draw, 0xE6 | stream << 8) alone, and the rule is one subtraction, one
// product and one addition per component, built without FMA contraction on either side, so the host twin (a serial
// loop over the same code) equals the kernel bit for bit at any num_worlds, shard or launch shape.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define DYNAMICS_THREADS 256
#define PURPOSE_ACCEL 0xE6u

struct DynamicsArgs {
    float lin_lo, lin_span, ang_lo, ang_span;   // limit = lo + span u; (0, 0) for a kind that is off
    float v_min, v_max, w_min, w_max, dt;
    uint32_t k0, k1, stream, draw, agent0;      // agent0: global index of row 0, world_offset * R
    bool lin_on, ang_on;
    size_t rows;
};

// what the tick executes for a command component x: |x| > 3e38 and NaN become 0 (rlca_env.cu's test), then the clip.
// The clip compares instead of calling fminf / fmaxf, so -0 passes unchanged on host and device alike.
__host__ __device__ __forceinline__ float tick_target(float x, float lo, float hi)
{
    if (!(fabsf(x) <= 3.0e38f)) x = 0.0f;
    return x < lo ? lo : (x > hi ? hi : x);
}

// one component under a limit: at most s = limit dt from prev, and the target itself when it is within reach
__host__ __device__ __forceinline__ float limited(float target, float prev, float s)
{
    const float d = target - prev;
    return d > s ? prev + s : (d < -s ? prev - s : target);
}

// the executed command of row a: a fresh row draws its limits and starts from rest, a crashed row starts from rest
__host__ __device__ __forceinline__ float2 dynamics_agent(const DynamicsArgs &q, size_t a, bool fresh, bool crashed,
                                                          float2 cmd, float2 *vel, float *lin, float *ang)
{
    float la, aa;
    if (fresh) {
        uint32_t c[4] = {q.agent0 + (uint32_t)a, q.draw, 0u, PURPOSE_ACCEL | (q.stream << 8)};
        dev_philox(c, q.k0, q.k1);
        la = q.lin_lo + q.lin_span * ((float)(c[0] >> 8) * 5.9604644775390625e-08f);
        aa = q.ang_lo + q.ang_span * ((float)(c[1] >> 8) * 5.9604644775390625e-08f);
        lin[a] = la;
        ang[a] = aa;
    } else {
        la = lin[a];
        aa = ang[a];
    }
    const float2 prev = (fresh || crashed) ? make_float2(0.0f, 0.0f) : vel[a];
    float2 e;
    e.x = tick_target(cmd.x, q.v_min, q.v_max);
    e.y = tick_target(cmd.y, q.w_min, q.w_max);
    if (q.lin_on) e.x = limited(e.x, prev.x, la * q.dt);
    if (q.ang_on) e.y = limited(e.y, prev.y, aa * q.dt);
    vel[a] = e;
    return e;
}

// One thread per agent: a float2 of command and of state in, a float2 of executed command and of state out.
__global__ void __launch_bounds__(DYNAMICS_THREADS)
    rlca_dynamics_action_kernel(DynamicsArgs q, const uchar4 *__restrict__ flags, const float2 *__restrict__ in,
                                float2 *__restrict__ out, float2 *__restrict__ vel, float *__restrict__ lin,
                                float *__restrict__ ang)
{
    const size_t a = (size_t)blockIdx.x * DYNAMICS_THREADS + threadIdx.x;
    if (a >= q.rows) return;
    bool fresh = true, crashed = false;
    if (flags != nullptr) {
        const uchar4 f = flags[a];
        fresh = f.w != 0;
        crashed = f.y != 0;
    }
    out[a] = dynamics_agent(q, a, fresh, crashed, in[a], vel, lin, ang);
}

// ------------------------------------------------------------------------------------------------ entries
// (0, 0) is off; anything else must be finite with 0 < lo <= hi <= RLCA_DYNAMICS_MAX_ACCEL (NaN fails every test)
static bool accel_range_ok(float lo, float hi)
{
    return (lo == 0.0f && hi == 0.0f) || (lo > 0.0f && lo <= hi && hi <= (float)RLCA_DYNAMICS_MAX_ACCEL);
}

static int dynamics_args(const rlca_env_config *cfg, const rlca_dynamics_params *p, const rlca_dynamics_state *st,
                         uint32_t draw, const float *in, const float *out, DynamicsArgs &q)
{
    if (!cfg || !p || !st) return rlca_set_err(RLCA_ERR_INVALID, "dynamics: cfg, params or state is NULL");
    if (!st->vel || !st->lin_limit || !st->ang_limit)
        return rlca_set_err(RLCA_ERR_INVALID, "dynamics: state vel, lin_limit or ang_limit is NULL");
    if (!in || !out) return rlca_set_err(RLCA_ERR_INVALID, "dynamics: action_in or action_out is NULL");
    if (cfg->robots_per_world < 1 || cfg->robots_per_world > RLCA_MAX_ROBOTS_PER_WORLD || cfg->num_worlds < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "dynamics: robots_per_world must be in 1..64 and num_worlds >= 1");
    if (cfg->world_offset < 0) return rlca_set_err(RLCA_ERR_INVALID, "dynamics: world_offset must be >= 0");
    if (!accel_range_ok(p->lin_lo, p->lin_hi) || !accel_range_ok(p->ang_lo, p->ang_hi))
        return rlca_set_err(RLCA_ERR_INVALID, "dynamics: every limit range must be (0, 0) or finite with "
                                              "0 < lo <= hi <= 100");
    if (p->stream_id >= (1u << 24)) return rlca_set_err(RLCA_ERR_INVALID, "dynamics: stream_id must be below 2^24");
    q.lin_lo = p->lin_lo;
    q.lin_span = p->lin_hi - p->lin_lo;
    q.ang_lo = p->ang_lo;
    q.ang_span = p->ang_hi - p->ang_lo;
    q.lin_on = p->lin_hi > 0.0f;
    q.ang_on = p->ang_hi > 0.0f;
    q.v_min = cfg->v_min;
    q.v_max = cfg->v_max;
    q.w_min = cfg->w_min;
    q.w_max = cfg->w_max;
    q.dt = cfg->dt;
    q.k0 = (uint32_t)p->seed;
    q.k1 = (uint32_t)(p->seed >> 32);
    q.stream = p->stream_id;
    q.draw = draw;
    q.agent0 = (uint32_t)cfg->world_offset * (uint32_t)cfg->robots_per_world;
    q.rows = (size_t)cfg->num_worlds * (size_t)cfg->robots_per_world;
    return RLCA_OK;
}

extern "C" int rlca_dynamics_action(const rlca_env_config *cfg, const rlca_dynamics_params *p,
                                    const rlca_dynamics_state *state, uint32_t draw, const unsigned char *flags_dev,
                                    const float *action_in_dev, float *action_out_dev, void *stream)
{
    DynamicsArgs q;
    int rc = dynamics_args(cfg, p, state, draw, action_in_dev, action_out_dev, q);
    if (rc) return rc;
    const unsigned grid = (unsigned)((q.rows + DYNAMICS_THREADS - 1) / DYNAMICS_THREADS);
    rlca_dynamics_action_kernel<<<grid, DYNAMICS_THREADS, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const uchar4 *>(flags_dev), reinterpret_cast<const float2 *>(action_in_dev),
        reinterpret_cast<float2 *>(action_out_dev), reinterpret_cast<float2 *>(state->vel), state->lin_limit,
        state->ang_limit);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_dynamics_action_host(const rlca_env_config *cfg, const rlca_dynamics_params *p,
                                         const rlca_dynamics_state *state, uint32_t draw,
                                         const unsigned char *flags_host, const float *action_in_host,
                                         float *action_out_host)
{
    DynamicsArgs q;
    int rc = dynamics_args(cfg, p, state, draw, action_in_host, action_out_host, q);
    if (rc) return rc;
    float2 *vel = reinterpret_cast<float2 *>(state->vel);
    for (size_t a = 0; a < q.rows; ++a) {
        const bool fresh = flags_host == nullptr || flags_host[4 * a + 3] != 0;
        const bool crashed = flags_host != nullptr && flags_host[4 * a + 1] != 0;
        const float2 e = dynamics_agent(q, a, fresh, crashed,
                                        make_float2(action_in_host[2 * a], action_in_host[2 * a + 1]), vel,
                                        state->lin_limit, state->ang_limit);
        action_out_host[2 * a] = e.x;
        action_out_host[2 * a + 1] = e.y;
    }
    return RLCA_OK;
}
