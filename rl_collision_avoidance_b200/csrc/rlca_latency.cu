// rlca_latency.cu — sensing and command latency around the tick (sm_90a), C ABI in include/rlca.h, DESIGN.md §9q.
//
// rlca_latency_scan replaces the newest frame of an observation stack, after a tick, with the true frame of d calls
// earlier, from a ring of the last scan_hi + 1 true frames per agent.  rlca_latency_action turns the command issued on
// a tick into the command issued l calls earlier, from a ring of the last cmd_hi + 1 commands per agent.  d and l are
// drawn per agent when it starts an episode and held until its next one.  Both are separate launches; the tick's
// kernels, its config and its outputs are untouched, and a run without latency issues neither.
//
// Latency is a file of its own, not a part of rlca_noise.cu, because it owns state across ticks: the rings and the
// per-episode delays.  Every delay is a function of (seed, global agent, draw, purpose | stream << 8) alone, and
// everything else is copies and integer arithmetic, so the host twins (serial loops over the same code) equal the
// kernels bit for bit at any num_worlds, shard or launch shape.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rlca.h"
#include "rlca_common.cuh"

#define LATENCY_THREADS 256
#define PURPOSE_SCAN_DELAY 0xE4u
#define PURPOSE_CMD_DELAY 0xE5u

struct LatencyArgs {
    uint32_t k0, k1, stream, draw, agent0;  // agent0: global index of row 0, world_offset * R
    uint32_t lo, span;                      // the kind's delay range: lo .. lo + span - 1
    uint32_t slots, slot;                   // ring slots (hi + 1) and the slot of this call, draw mod slots
    int beams, groups;                      // groups = ceil(beams / 4)
    size_t rows;
};

// the delay of `agent` drawn at this call: lo + floor(span w0 / 2^32), w0 the first Philox word of
// (agent, draw, 0, purpose | stream << 8)
__host__ __device__ __forceinline__ uint8_t latency_delay(const LatencyArgs &q, uint32_t agent, uint32_t purpose)
{
    uint32_t c[4] = {agent, q.draw, 0u, purpose | (q.stream << 8)};
    dev_philox(c, q.k0, q.k1);
    return (uint8_t)(q.lo + (uint32_t)(((uint64_t)q.span * (uint64_t)c[0]) >> 32));
}

// the ring slot read by an agent of delay d at this call: (draw - d) mod slots, d < slots
__host__ __device__ __forceinline__ uint32_t latency_read_slot(const LatencyArgs &q, uint32_t d)
{
    return q.slot >= d ? q.slot - d : q.slot + q.slots - d;
}

// element (row, group) of the scan pass, scalar loads: `stack` is the row's three frames, `ring` its slots frames
__host__ __device__ __forceinline__ void scan_group(const LatencyArgs &q, size_t row, int g, bool fresh, float *stack,
                                                    float *ring, uint8_t *delay)
{
    const int B = q.beams, b0 = 4 * g, n = B - b0 < 4 ? B - b0 : 4;
    float *newest = stack + 2 * (size_t)B + b0;
    if (fresh) {                                // every slot holds the first frame; the stack already does
        for (uint32_t s = 0; s < q.slots; ++s)
            for (int j = 0; j < n; ++j) ring[s * (size_t)B + b0 + j] = newest[j];
        if (g == 0) delay[row] = latency_delay(q, q.agent0 + (uint32_t)row, PURPOSE_SCAN_DELAY);
        return;
    }
    const uint32_t rs = latency_read_slot(q, delay[row]);
    float *w = ring + q.slot * (size_t)B + b0;
    const float *r = ring + rs * (size_t)B + b0;
    for (int j = 0; j < n; ++j) w[j] = newest[j];
    for (int j = 0; j < n; ++j) newest[j] = r[j];
}

// the executed command of agent a: ring slot `slot` gets the issued command, the command of delay l's slot leaves
__host__ __device__ __forceinline__ float2 command_agent(const LatencyArgs &q, size_t a, bool fresh, float2 cmd,
                                                         float2 *ring, uint8_t *delay)
{
    uint32_t l;
    if (fresh) {                                // a new episode: every slot holds its first command (DESIGN.md §9q)
        for (uint32_t s = 0; s < q.slots; ++s) ring[s] = cmd;
        l = latency_delay(q, q.agent0 + (uint32_t)a, PURPOSE_CMD_DELAY);
        delay[a] = (uint8_t)l;
    } else {
        l = delay[a];
    }
    ring[q.slot] = cmd;
    return ring[latency_read_slot(q, l)];
}

// One thread per (row, group of four beams).  VEC: beams % 4 == 0 and a 16-byte aligned stack and ring, one float4 per
// frame.  The group-0 thread of a fresh row draws its delay; the row's other threads never read it.
template <bool VEC>
__global__ void __launch_bounds__(LATENCY_THREADS)
    rlca_latency_scan_kernel(LatencyArgs q, const uchar4 *__restrict__ flags, float *__restrict__ stack,
                             float *__restrict__ ring, uint8_t *__restrict__ delay)
{
    const size_t t = (size_t)blockIdx.x * LATENCY_THREADS + threadIdx.x;
    if (t >= q.rows * (size_t)q.groups) return;
    const size_t row = t / (size_t)q.groups;
    const int g = (int)(t - row * (size_t)q.groups);
    const bool fresh = flags == nullptr || flags[row].w != 0;
    float *s = stack + row * 3 * (size_t)q.beams;
    float *rg = ring + row * (size_t)q.slots * (size_t)q.beams;
    if (VEC) {
        const int G = q.groups;
        float4 *s4 = reinterpret_cast<float4 *>(s) + 2 * G + g;
        float4 *r4 = reinterpret_cast<float4 *>(rg) + g;
        const float4 o = *s4;
        if (fresh) {
            for (uint32_t k = 0; k < q.slots; ++k) r4[k * (size_t)G] = o;
            if (g == 0) delay[row] = latency_delay(q, q.agent0 + (uint32_t)row, PURPOSE_SCAN_DELAY);
            return;
        }
        const uint32_t rs = latency_read_slot(q, delay[row]);
        r4[q.slot * (size_t)G] = o;
        *s4 = r4[rs * (size_t)G];
    } else {
        scan_group(q, row, g, fresh, s, rg, delay);
    }
}

__global__ void __launch_bounds__(LATENCY_THREADS)
    rlca_latency_action_kernel(LatencyArgs q, const uchar4 *__restrict__ flags, const float2 *__restrict__ in,
                               float2 *__restrict__ out, float2 *__restrict__ ring, uint8_t *__restrict__ delay)
{
    const size_t a = (size_t)blockIdx.x * LATENCY_THREADS + threadIdx.x;
    if (a >= q.rows) return;
    const bool fresh = flags == nullptr || flags[a].w != 0;
    out[a] = command_agent(q, a, fresh, in[a], ring + a * (size_t)q.slots, delay);
}

// ------------------------------------------------------------------------------------------------ entries
static bool delay_range_ok(int32_t lo, int32_t hi) { return lo >= 0 && lo <= hi && hi <= RLCA_LATENCY_MAX_DELAY; }

// the arguments of one kind (scan: lo, hi = scan_lo, scan_hi; command: cmd_lo, cmd_hi) at call `draw`
static int latency_args(const rlca_env_config *cfg, const rlca_latency_params *p, const rlca_latency_state *st,
                        bool scan, uint32_t draw, LatencyArgs &q)
{
    if (!cfg || !p || !st) return rlca_set_err(RLCA_ERR_INVALID, "latency: cfg, params or state is NULL");
    if (cfg->robots_per_world < 1 || cfg->robots_per_world > RLCA_MAX_ROBOTS_PER_WORLD || cfg->num_worlds < 1)
        return rlca_set_err(RLCA_ERR_INVALID, "latency: robots_per_world must be in 1..64 and num_worlds >= 1");
    if (cfg->beams < 1 || cfg->world_offset < 0)
        return rlca_set_err(RLCA_ERR_INVALID, "latency: beams must be >= 1 and world_offset >= 0");
    if (!delay_range_ok(p->scan_lo, p->scan_hi) || !delay_range_ok(p->cmd_lo, p->cmd_hi))
        return rlca_set_err(RLCA_ERR_INVALID, "latency: every delay range must satisfy 0 <= lo <= hi <= 8 ticks");
    if (p->stream_id >= (1u << 24)) return rlca_set_err(RLCA_ERR_INVALID, "latency: stream_id must be below 2^24");
    const int32_t lo = scan ? p->scan_lo : p->cmd_lo, hi = scan ? p->scan_hi : p->cmd_hi;
    if (hi > 0 && (scan ? (!st->scan_ring || !st->scan_delay) : (!st->cmd_ring || !st->cmd_delay)))
        return rlca_set_err(RLCA_ERR_INVALID, scan ? "latency: scan_ring or scan_delay is NULL"
                                                   : "latency: cmd_ring or cmd_delay is NULL");
    q.k0 = (uint32_t)p->seed;
    q.k1 = (uint32_t)(p->seed >> 32);
    q.stream = p->stream_id;
    q.draw = draw;
    q.agent0 = (uint32_t)cfg->world_offset * (uint32_t)cfg->robots_per_world;
    q.lo = (uint32_t)lo;
    q.span = (uint32_t)(hi - lo + 1);
    q.slots = (uint32_t)hi + 1u;
    q.slot = draw % q.slots;
    q.beams = cfg->beams;
    q.groups = (cfg->beams + 3) / 4;
    q.rows = (size_t)cfg->num_worlds * (size_t)cfg->robots_per_world;
    return RLCA_OK;
}

static unsigned blocks(size_t threads) { return (unsigned)((threads + LATENCY_THREADS - 1) / LATENCY_THREADS); }

extern "C" int rlca_latency_scan(const rlca_env_config *cfg, const rlca_latency_params *p,
                                 const rlca_latency_state *state, uint32_t draw, const unsigned char *flags_dev,
                                 float *stack_dev, void *stream)
{
    LatencyArgs q;
    int rc = latency_args(cfg, p, state, true, draw, q);
    if (rc) return rc;
    if (!stack_dev) return rlca_set_err(RLCA_ERR_INVALID, "rlca_latency_scan: stack_dev is NULL");
    if (p->scan_hi == 0) return RLCA_OK;        // no scan delay: the stack is what the robot reads
    const uchar4 *flags = reinterpret_cast<const uchar4 *>(flags_dev);
    const unsigned grid = blocks(q.rows * (size_t)q.groups);
    const bool vec = (q.beams & 3) == 0 && ((reinterpret_cast<uintptr_t>(stack_dev) |
                                             reinterpret_cast<uintptr_t>(state->scan_ring)) & 15) == 0;
    if (vec)
        rlca_latency_scan_kernel<true><<<grid, LATENCY_THREADS, 0, (cudaStream_t)stream>>>(
            q, flags, stack_dev, state->scan_ring, state->scan_delay);
    else
        rlca_latency_scan_kernel<false><<<grid, LATENCY_THREADS, 0, (cudaStream_t)stream>>>(
            q, flags, stack_dev, state->scan_ring, state->scan_delay);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_latency_action(const rlca_env_config *cfg, const rlca_latency_params *p,
                                   const rlca_latency_state *state, uint32_t draw, const unsigned char *flags_dev,
                                   const float *action_in_dev, float *action_out_dev, void *stream)
{
    LatencyArgs q;
    int rc = latency_args(cfg, p, state, false, draw, q);
    if (rc) return rc;
    if (!action_in_dev || !action_out_dev)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_latency_action: action_in_dev or action_out_dev is NULL");
    if (p->cmd_hi == 0) {                       // no command latency: the issued command is executed
        if (action_out_dev != action_in_dev)
            RLCA_CUDA_TRY(cudaMemcpyAsync(action_out_dev, action_in_dev, q.rows * 2 * sizeof(float),
                                          cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
        return RLCA_OK;
    }
    rlca_latency_action_kernel<<<blocks(q.rows), LATENCY_THREADS, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const uchar4 *>(flags_dev), reinterpret_cast<const float2 *>(action_in_dev),
        reinterpret_cast<float2 *>(action_out_dev), reinterpret_cast<float2 *>(state->cmd_ring), state->cmd_delay);
    RLCA_CUDA_TRY(cudaGetLastError());
    return RLCA_OK;
}

extern "C" int rlca_latency_scan_host(const rlca_env_config *cfg, const rlca_latency_params *p,
                                      const rlca_latency_state *state, uint32_t draw,
                                      const unsigned char *flags_host, float *stack_host)
{
    LatencyArgs q;
    int rc = latency_args(cfg, p, state, true, draw, q);
    if (rc) return rc;
    if (!stack_host) return rlca_set_err(RLCA_ERR_INVALID, "rlca_latency_scan_host: stack_host is NULL");
    if (p->scan_hi == 0) return RLCA_OK;
    for (size_t row = 0; row < q.rows; ++row) {
        const bool fresh = flags_host == nullptr || flags_host[4 * row + 3] != 0;
        for (int g = 0; g < q.groups; ++g)
            scan_group(q, row, g, fresh, stack_host + row * 3 * (size_t)q.beams,
                       state->scan_ring + row * (size_t)q.slots * (size_t)q.beams, state->scan_delay);
    }
    return RLCA_OK;
}

extern "C" int rlca_latency_action_host(const rlca_env_config *cfg, const rlca_latency_params *p,
                                        const rlca_latency_state *state, uint32_t draw,
                                        const unsigned char *flags_host, const float *action_in_host,
                                        float *action_out_host)
{
    LatencyArgs q;
    int rc = latency_args(cfg, p, state, false, draw, q);
    if (rc) return rc;
    if (!action_in_host || !action_out_host)
        return rlca_set_err(RLCA_ERR_INVALID, "rlca_latency_action_host: action_in_host or action_out_host is NULL");
    float2 *ring = reinterpret_cast<float2 *>(state->cmd_ring);
    for (size_t a = 0; a < q.rows; ++a) {
        const float2 cmd = make_float2(action_in_host[2 * a], action_in_host[2 * a + 1]);
        float2 e = cmd;
        if (p->cmd_hi > 0) {
            const bool fresh = flags_host == nullptr || flags_host[4 * a + 3] != 0;
            e = command_agent(q, a, fresh, cmd, ring + a * (size_t)q.slots, state->cmd_delay);
        }
        action_out_host[2 * a] = e.x;
        action_out_host[2 * a + 1] = e.y;
    }
    return RLCA_OK;
}
