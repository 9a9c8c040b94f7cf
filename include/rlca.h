/*
 * rlca.h — C ABI of the H100-native collision-avoidance hot path (librlca.so).
 *
 * Drop-in boundary for the path BASELINE.json's north_star names.  The
 * reference has no FFI of its own (its seam is duck-typed Python over ROS
 * topics, SURVEY.md §8(b)); each entry point below states the reference
 * interface it replaces (file:line in the reference).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only; no torch / C++ types.
 *   - Every function returns int: 0 = RLCA_OK, otherwise an rlca_status;
 *     the message is available from rlca_last_error() (thread-local).
 *   - Pointers named *_dev are DEVICE pointers owned by the caller (PyTorch
 *     allocates them); the library never frees them.  `stream` is a
 *     cudaStream_t passed as void* (NULL = legacy default stream).  Calls are
 *     asynchronous on that stream unless the name ends in _host.
 *   - A handle is bound to the CUDA device current at creation, owns only the
 *     uploaded static map, scenario tables and the beam table, and is not
 *     thread-safe.  Different handles are independent.
 *   - There is no CPU fallback: without a CUDA device every call fails loudly.
 */
#ifndef RLCA_H
#define RLCA_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum rlca_status {
    RLCA_OK = 0,
    RLCA_ERR_INVALID = 1,     /* bad argument / config */
    RLCA_ERR_CUDA = 2,        /* CUDA runtime error (sticky errors surface here) */
    RLCA_ERR_UNSUPPORTED = 3, /* e.g. map too large for the shared-memory owner grid */
    RLCA_ERR_NO_DEVICE = 4
} rlca_status;

#define RLCA_MAX_ROBOTS_PER_WORLD 64

/* Scenario + geometry.  Field meanings and reference sources:
 *   robots_per_world  24/44/50 agents per world   worlds/stage1.world:107-130, stage2.world:113-165, circle.world:106-155
 *   beams / raw_beams beam_num / sensor samples   stage_world1.py:17,126-139 ; worlds/stage1.world:14
 *   resolution        cell size                   worlds/stage1.world:3
 *   dt                0.1 s tick                  default interval_sim; test/hztest.xml:14,18
 *   range_max, fov    6.0 m, pi                   worlds/stage1.world:12-13
 *   half_len/half_wid 0.22, 0.19                  worlds/stage1.world:83
 *   goal_radius ... w_penalty                     stage_world1.py:34,183-204 ; circle_world.py:195
 *   v_min..w_max      action bound                ppo_stage1.py:170
 *   timeout           150/200/10000               stage_world1.py:206, stage_world2.py:203, circle_world.py:198
 *   pre_distance_zero quirk                       stage_world2.py:170, circle_world.py:166
 *   scenario          0 = stage1 random spawn/goal (stage_world1.py:251-274)
 *                     1 = stage2 tables + random region for flagged rows (stage_world2.py:164-171,210-221,250-287)
 *                     2 = circle tables (circle_world.py:164-167,205-208)
 */
typedef struct rlca_env_config {
    int32_t robots_per_world;
    int32_t num_worlds;          /* worlds on THIS device (shard) */
    int32_t beams;
    int32_t raw_beams;
    int32_t grid_w, grid_h;      /* static map cells; grid_w is also the row pitch */
    int32_t origin_cx, origin_cy;/* cell index of world (0,0): cell = floor(x*ppm) + origin */
    float resolution;
    float ppm;
    float dt;
    float inv_dt;
    float range_max;
    float range_cells;           /* ppm * range_max */
    float fov;
    float half_len, half_wid;
    float goal_radius;
    float reward_arrive;
    float reward_collision;
    float progress_gain;
    float w_threshold;
    float w_penalty;
    float v_min, v_max, w_min, w_max;
    int32_t timeout;
    int32_t pre_distance_zero;
    int32_t scenario;
    int32_t auto_reset;          /* 0 = caller resets; 1 = a done agent is re-spawned inside the tick (stage 1,
                                  * ppo_stage1.py:50-53); 2 = group-synchronous (stage 2): a done agent idles on its last
                                  * command until every robot of its group (goal_tab[r][3] = group id) is done, then the
                                  * whole group is re-spawned (ppo_stage2.py:72-84,105-106; model/utils.py:81-87) */
    int32_t max_reject;          /* cap on rejection-sampling tries */
    int32_t world_offset;        /* global index of this shard's first world (RNG keys are global) */
    uint64_t seed;
} rlca_env_config;

/* Per-agent simulator state, N = robots_per_world * num_worlds rows of 4 x 32 bit:
 *   pose  x, y, theta, distance-to-goal after the last tick (= pre_distance next tick)
 *   goal  goal_x, goal_y, last commanded v, last commanded w (odom twist, stageros.cpp:547-550)
 *   acc   episode reward, last reward, init_x, init_y
 *   meta  step counter t, episode index, stall flag (is_crashed, stageros.cpp:560-564), terminal latch */
typedef struct rlca_env_state {
    float *pose_dev;
    float *goal_dev;
    float *acc_dev;
    int32_t *meta_dev;
} rlca_env_state;

/* Inputs / outputs of one tick.  obs may point into a rollout buffer slice.
 *   action (N,2) raw policy action (clipped inside)          model/ppo.py:73-75, stage_world1.py:226-234
 *   live   (N) u8 or NULL; 0 = agent idles on its last command  ppo_stage2.py:72-84
 *   obs    (N,beams) scan/6 - 0.5                             stage_world1.py:122-140
 *   reward (N)  flags (N,4) u8 = done, crashed, result{0,1 Reach Goal,2 Crashed,3 Time out}, was_reset
 *   gs     (N,4) local goal x,y + speed v,w                   stage_world1.py:143-144,155-160
 *   eplog  (N,8) written for agents whose episode ended: goal_x, goal_y, ep_reward, steps,
 *          init_x, init_y, result, episode                    ppo_stage1.py:127-131 */
typedef struct rlca_step_io {
    const float *action_dev;
    const uint8_t *live_dev;
    float *obs_dev;
    float *reward_dev;
    uint8_t *flags_dev;
    float *gs_dev;
    float *eplog_dev;
    const float *stack_in_dev;   /* optional (N,3,beams) scan FIFO (ppo_stage1.py:60,87-89): */
    float *stack_out_dev;        /*   out = [in[1], in[2], new scan], or 3 x new scan after a re-spawn; both or neither */
} rlca_step_io;

/* Host-side walk tables of the table-driven lidar for a given range_cells = range_max / resolution (no device
 * needed; the same code rlca_env_set_map runs, exported so that CPU tests can check it against the cell-by-cell
 * walk of World::Raytrace, SURVEY App. A.7).  Slots = the truncated end points (trunc(R cos a), trunc(R sin a)) any
 * ray can have.  Call with NULL buffers for the sizes, then with
 *   slot_keys   [2 * nslots] int16  (idx, idy) of every slot, ordered by angle
 *   keyslot     [(2 kr + 1)^2] uint16  (idy + kr) * (2 kr + 1) + (idx + kr) -> slot, 0xffff = cannot occur
 *   inv_off     [(2 kr + 1)^2 + 1], inv_ent [nentries]: per relative cell, slot | dominant-axis distance << 16 of
 *               every walk that tests that cell. */
int rlca_walk_tables_host(float range_cells, int32_t *kr, int32_t *nslots, int32_t *nentries, int16_t *slot_keys,
                          uint16_t *keyslot, uint32_t *inv_off, uint32_t *inv_ent);

/* The same inverse lists as the small-map lidar reads them when the range has at most 255 slots (RLCA_ERR_UNSUPPORTED
 * otherwise).  Call with NULL buffers for the sizes, then with
 *   records   [4 * nrecords] uint32, one 16-byte record per relative cell (nrecords = (2 kr + 1)^2):
 *             word 0 = list length (bits 0-7) | offset of the list's 7th entry in `overflow` (bits 8-31),
 *             words 1-3 = entries 0-5, two per word (the even entry in the low half)
 *   overflow  [noverflow] uint16, entries 6, 7, ... of every list, lists in relative-cell order
 * An entry is slot | dominant-axis distance << 8; the order of a list is that of inv_ent. */
int rlca_inv_records_host(float range_cells, int32_t *nrecords, int32_t *noverflow, uint32_t *records,
                          uint16_t *overflow);

typedef struct rlca_env rlca_env;

/* Replaces StageNode construction + world->Load (stageros.cpp:311-355): creates the
 * device-side world for a batch of identical worlds. */
int rlca_env_create(const rlca_env_config *cfg, rlca_env **out);
int rlca_env_destroy(rlca_env *env);

/* Upload the static occupancy grid (HOST pointer, grid_h*grid_w bytes, 0 = free,
 * non-zero = obstacle).  Replaces libstage's bitmap/polygon block rasterisation at load
 * (worlds/stage1.world:43-49, stage2.world:169-297). */
int rlca_env_set_map(rlca_env *env, const uint8_t *cells_host, int32_t grid_w, int32_t grid_h);

/* Scenario tables (HOST pointers, robots_per_world rows of 4 floats):
 *   init_tab  x, y, theta, random_flag   (world-file agent poses / model/utils.py:6-25,41-53)
 *   goal_tab  gx, gy, random_flag, group id   (model/utils.py:27-38,55-63,83) */
int rlca_env_set_tables(rlca_env *env, const float *init_tab_host, const float *goal_tab_host);

/* reset_world (stage_world1.py:162-169 -> cb_reset_srv stageros.cpp:260-269) when
 * clear_world == 1, then reset_pose + generate_goal_point (stage_world1.py:171-177,213-223)
 * for agents with mask != 0 (mask_dev NULL = all agents).  In place.
 * clear_world == 2: generate_goal_point ALONE for the masked agents (stage_world1.py:171-177 ->
 * generate_random_goal :262-274): a goal for the CURRENT pose from the draws of the current episode,
 * pre_distance / init_pose refreshed, pose and counters untouched. */
int rlca_env_reset(rlca_env *env, const rlca_env_state *state, const uint8_t *mask_dev,
                   int32_t clear_world, void *stream);

/* Scan / local goal / speed from the current poses without ticking
 * (get_laser_observation, get_local_goal, get_self_speed right after a reset:
 * ppo_stage1.py:59-63).  io->obs_dev and io->gs_dev are written. */
int rlca_env_observe(rlca_env *env, const rlca_env_state *state, const rlca_step_io *io, void *stream);

/* ONE fused tick over the whole agent batch: control_vel (stage_world1.py:226-234) ->
 * World::UpdateAll (stageros.cpp:448: integrate, collide, stall) -> WorldCallback
 * (stageros.cpp:451-611: GT velocity, is_crashed) -> get_reward_and_terminate
 * (stage_world1.py:180-211) -> optional re-spawn -> lidar raytrace from the final pose
 * (stageros.cpp:479-516) -> get_laser_observation / get_local_goal / get_self_speed.
 * Reads state_in, writes state_out (they may alias only when the launch uses one CTA
 * per world; pass distinct buffers and swap them each tick otherwise). */
int rlca_env_step(rlca_env *env, const rlca_env_state *state_in, const rlca_env_state *state_out,
                  const rlca_step_io *io, void *stream);

/* Same tick driven from HOST buffers (the reference-facing call: actions arrive from
 * the host, observations/rewards/flags return to it), ending with a stream synchronize.
 * Any *_host may be NULL to skip it.  io holds the device buffers, which are written as
 * by rlca_env_step (except action_dev in the zero-copy modes).  Host traffic, see
 * rlca_env_set_host_zero_copy:
 *   1 (default) pinned host buffers are used through their device-mapped aliases: the
 *               kernel reads action_host and mirrors reward/flags/gs and every scan to
 *               host memory with posted PCIe writes while it runs - no DMA operation at
 *               all in the call;
 *   2           the same for the small buffers, the scans (4*beams of the 4*beams + 24
 *               bytes an agent returns) cross by DMA: the shard is ticked in `host chunks`
 *               world ranges and each range's scans are copied on an internal stream
 *               while the next range is ticked;
 *   0           DMA copies only (H2D, tick in world ranges, D2H).
 * Pageable host buffers and the global-grid path fall back to mode 0.  Results are
 * identical in every mode (worlds are independent). */
int rlca_env_step_host(rlca_env *env, const rlca_env_state *state_in, const rlca_env_state *state_out,
                       const rlca_step_io *io, const float *action_host, float *obs_host,
                       float *reward_host, uint8_t *flags_host, float *gs_host, void *stream);

/* Stand-alone lidar raycast (World::Raytrace via ModelRanger, stageros.cpp:479-516):
 * pose_dev (N,4) x,y,theta,_ -> ranges_dev (N,beams) in metres (normalise = 0) or
 * scan/6-0.5 (normalise = 1).  Other robots' footprints are seen, own is excluded. */
int rlca_raycast(rlca_env *env, const float *pose_dev, float *ranges_dev, int32_t normalise, void *stream);

/* World ranges per rlca_env_step_host call on the DMA path: 0 = library default (2),
 * 1 = strictly serial (copy in, one launch, copy out), up to 16. */
int rlca_env_set_host_chunks(rlca_env *env, int32_t chunks);
/* Host traffic mode of rlca_env_step_host: 0, 1 or 2 (see there); -1 = back to the library default. */
int rlca_env_set_host_zero_copy(rlca_env *env, int32_t mode);

/* Launch shape knob: CTAs per world (>= 1).  0 = library default (auto). */
int rlca_env_set_ctas_per_world(rlca_env *env, int32_t ctas_per_world);
/* Number of kernels the library launched on behalf of this handle so far. */
int64_t rlca_env_launch_count(const rlca_env *env);
/* Small maps: CTAs of the tick's lidar launch that one SM holds at once (its shared memory and registers at the
 * map's tables); 0 for a big map.  The launch is sized for 8. */
int rlca_env_lidar_ctas_per_sm(const rlca_env *env, int32_t *ctas);


/* =====================================================================================
 * Learning half: CNNPolicy forward/backward, PPO loss, GAE, Adam.
 * Replaces the PyTorch library calls of model/net.py:37-80 and model/ppo.py:122-194.
 *
 * Parameters live in ONE flat fp32 buffer of RLCA_POLICY_NPARAMS floats laid out in the
 * order of the reference's state_dict (model/net.py:16-34; SURVEY.md App. C):
 *   logstd(2) | act_fea_cv1.w(32,3,5) .b(32) | act_fea_cv2.w(32,32,3) .b(32) | act_fc1.w(256,4096) .b(256)
 *   | act_fc2.w(128,260) .b(128) | actor1.w(1,128) .b(1) | actor2.w(1,128) .b(1)
 *   | crt_fea_cv1 ... crt_fc2 (same shapes) | critic.w(1,128) .b(1)
 * rlca_policy_param_offset(i) returns the float offset of tensor i (0..22) in that order,
 * and i == 23 returns the total.  Gradients and Adam moments use the same layout, so the
 * optimizer is one fused elementwise kernel and the data-parallel all-reduce one buffer.
 * ===================================================================================== */
#define RLCA_POLICY_NPARAMS 2172101
#define RLCA_POLICY_NTENSORS 23
#define RLCA_OBS_FRAMES 3
#define RLCA_OBS_BEAMS 512

typedef struct rlca_policy rlca_policy;   /* workspace (activations kept for backward) */

int64_t rlca_policy_param_offset(int32_t tensor_index);
int64_t rlca_policy_param_size(int32_t tensor_index);     /* unpadded element count of tensor i */
int64_t rlca_policy_launch_count(const rlca_policy *pol);

/* Data-parallel overlap hook (model/ppo.py:186-188 takes an optimizer step per minibatch, so the gradient all-reduce is
 * on the critical path): `event` (a cudaEvent_t, or NULL to clear) is recorded by every rlca_policy_backward on its
 * stream as soon as all gradients OUTSIDE the two conv towers are final - fc1/fc2/heads, 97 % of the flat buffer,
 * tensors 5..12 and 17..22 of the state_dict order.  The caller all-reduces those ranges on another stream while the
 * dF GEMM and the conv tower backward are still running, and the conv ranges afterwards. */
int rlca_policy_set_grad_event(rlca_policy *pol, void *event);

/* Data-parallel optimizer step fused with its collective over NVLink peer memory (csrc/rlca_dp.cu): reduce-scatter of
 * the gradient + Adam + all-gather of the parameter and both moments in ONE kernel.  *_ptrs are HOST arrays of `world`
 * device addresses: the peer mappings of every rank's flat gradient / parameter / exp_avg / exp_avg_sq buffer (n floats
 * each, n % 4 == 0), e.g. from a symmetric-memory allocation; mc_* are the NVSwitch multicast mappings of the same
 * buffers (NVLS: multimem.ld_reduce / multimem.st) or 0 to use plain peer loads and stores.  Rank r updates elements
 * [r * ceil(n / world), ...): the new parameters go into every rank's buffer (replicated bit for bit), the two
 * moments stay in the owner's buffer (sharded optimizer state; a checkpoint reads the shards back through the peer
 * mappings) unless replicate_moments != 0.  The caller puts a cross-GPU barrier before (all gradients written) and
 * after (all shards written) the call.  Same arithmetic as rlca_adam_step with grad_scale = 1 / world on the summed gradient
 * (model/ppo.py:186-188 + ppo_stage1.py:179 at any world size). */
int rlca_adam_step_allreduce(const uint64_t *grad_ptrs, const uint64_t *param_ptrs, const uint64_t *m_ptrs,
                             const uint64_t *v_ptrs, uint64_t mc_grad, uint64_t mc_param, uint64_t mc_m, uint64_t mc_v,
                             int32_t rank, int32_t world, int64_t n, float lr, float beta1, float beta2, float eps,
                             int32_t step, float grad_scale, int32_t replicate_moments, void *stream);
/* Conv tower + fc1 forward/backward GEMMs on the Hopper tensor cores (wgmma) with 3xTF32 error compensation
 * (enable = 1, the default); 2 = fc1 GEMMs only; 0 selects the plain fp32 CUDA-core kernels (kept as the
 * cross-check for the tensor-core path). */
int rlca_policy_set_tensor_cores(rlca_policy *pol, int32_t enable);
/* Copies the conv-tower features of the last forward, relu(conv2) flattened as c*128+q (model/net.py:42-44 `a.view`),
 * tower 0 = actor, 1 = critic, into dst_dev (nb x 4096 floats).  Inspection hook for the parity tests. */
int rlca_policy_features(const rlca_policy *pol, int32_t tower, int32_t nb, float *dst_dev, void *stream);
/* Tell the workspace that params_dev changed (optimizer step, checkpoint load): derived copies of the weights
 * (tf32 hi/lo splits, transposes) are rebuilt at the next forward.  A fresh workspace starts dirty. */
int rlca_policy_weights_changed(rlca_policy *pol);

/* Workspace sized for batches up to max_batch rows. */
int rlca_policy_create(int32_t max_batch, rlca_policy **out);
int rlca_policy_destroy(rlca_policy *pol);

/* CNNPolicy.forward without sampling (model/net.py:37-70): obs (nb,3,512), gs (nb,4) =
 * local goal x,y + speed v,w  ->  value (nb), mean (nb,2).  Activations stay in the
 * workspace for rlca_policy_backward. */
int rlca_policy_forward(rlca_policy *pol, const float *params_dev, const float *obs_dev, const float *gs_dev,
                        int32_t nb, float *value_dev, float *mean_dev, void *stream);

/* action ~ N(mean, exp(logstd)) with a counter-based generator (replaces torch.normal,
 * model/net.py:53-55), logprob = log_normal_density summed over the 2 dims
 * (model/utils.py:90-97), scaled = clip(action, [v_min,w_min], [v_max,w_max]) (model/ppo.py:75).
 * deterministic == 0 -> row i draws Philox4x32-10 of counter (i, counter lo, counter hi, 0x5A17) under key
 *   (seed lo, seed hi); u1 = ((w0 >> 8) + 1) * 2^-24, u2 = (w1 >> 8) * 2^-24, Box-Muller z = sqrt(-2 ln u1) *
 *   (cos, sin)(2 pi u2) and action = mean + exp(logstd) * z.  A row's draw depends on (seed, counter, i) only;
 * deterministic == 1 -> action = mean (generate_action_no_sampling, model/ppo.py:84-107);
 * deterministic == 2 -> action_dev is an INPUT and only its logprob is evaluated (evaluate_actions, model/net.py:72-80).
 * Any other deterministic, nb < 1 or a NULL params, mean, action or logprob -> RLCA_ERR_INVALID, nothing launched.
 * scaled_dev may be NULL. */
int rlca_policy_sample(const float *params_dev, const float *mean_dev, int32_t nb, uint64_t seed, uint64_t counter,
                       int32_t deterministic, float *action_dev, float *logprob_dev, float *scaled_dev, void *stream);

/* Clipped-surrogate + value + entropy loss of one minibatch and its gradient w.r.t. the
 * network outputs (model/ppo.py:172-185): loss = -mean(min(r*A, clamp(r,1-c,1+c)*A))
 * + value_coef*MSE(V,target) - coeff_entropy*entropy.  losses_dev[0..2] = policy_loss,
 * value_loss, entropy (the three numbers logged to ppo.log, model/ppo.py:189-192).  The output
 * gradients stay in the workspace for rlca_policy_backward. */
int rlca_ppo_loss_fwd_bwd(rlca_policy *pol, const float *params_dev, const float *value_dev, const float *mean_dev,
                          const float *action_dev, const float *old_logprob_dev, const float *adv_dev,
                          const float *target_dev, int32_t nb, float clip_value, float coeff_entropy,
                          float value_coef, float *losses_dev, void *stream);

/* Same, with every gradient multiplied by grad_weight (the logged losses are not).  Data-parallel training: a rank
 * whose minibatch holds nb_r of the step's sum(nb_r) rows passes grad_weight = nb_r * world_size / sum(nb_r), so that
 * the all-reduced gradient / world_size is the mean over ALL rows of the global minibatch (the reference's single
 * process sees one batch, model/ppo.py:172-188). */
int rlca_ppo_loss_fwd_bwd_weighted(rlca_policy *pol, const float *params_dev, const float *value_dev,
                                   const float *mean_dev, const float *action_dev, const float *old_logprob_dev,
                                   const float *adv_dev, const float *target_dev, int32_t nb, float clip_value,
                                   float coeff_entropy, float value_coef, float grad_weight, float *losses_dev,
                                   void *stream);

/* PPO update diagnostics (DESIGN.md §9n): what an update did to the policy and the critic, accumulated on the device
 * into rows of RLCA_PPO_DIAG_COLUMNS doubles, one row per epoch, read back once per update.  Every column has ONE merge
 * rule - sum, max or min - by which minibatches, epochs and data-parallel ranks combine.  A fresh row holds 0 in the
 * sum columns, -inf in the max columns and +inf in the min column.  With r = exp(new_lp - old_lp), A the advantage, t
 * the value target, V the value and c the clip value: */
#define RLCA_PPO_DIAG_N 0               /* rows */
#define RLCA_PPO_DIAG_SUM_KL 1          /* sum of old_lp - new_lp */
#define RLCA_PPO_DIAG_SUM_KL_K3 2       /* sum of (r - 1) - log r, with r - 1 as expm1(log r) */
#define RLCA_PPO_DIAG_CLIPPED 3         /* rows with |r - 1| > c */
#define RLCA_PPO_DIAG_CUT 4             /* rows whose surrogate gradient is cut: r > 1 + c with A > 0, r < 1 - c with A < 0 */
#define RLCA_PPO_DIAG_SUM_RATIO 5       /* sum of r */
#define RLCA_PPO_DIAG_SUM_ERR 6         /* sum, sum of squares (6, 7) of t - V */
#define RLCA_PPO_DIAG_SUM_TARGET 8      /* sum, sum of squares (8, 9) of t */
#define RLCA_PPO_DIAG_SUM_VALUE 10      /* sum of V */
#define RLCA_PPO_DIAG_SUM_ADV 11        /* sum, sum of squares (11, 12) of A */
#define RLCA_PPO_DIAG_MEAN_OUT 13       /* rows whose policy mean lies outside the action bound, per action dimension (13, 14) */
#define RLCA_PPO_DIAG_ACTION_OUT 15     /* rows whose sampled action lies outside it (15, 16) */
#define RLCA_PPO_DIAG_MAX_RATIO 17      /* MAX: largest r */
#define RLCA_PPO_DIAG_MIN_RATIO 18      /* MIN: smallest r */
#define RLCA_PPO_DIAG_GRAD_STEPS 19     /* rlca_grad_sumsq calls */
#define RLCA_PPO_DIAG_GRAD_SUMSQ 20     /* sum of g^2 of each of the RLCA_POLICY_NTENSORS tensors (20 .. 42) */
#define RLCA_PPO_DIAG_MAX_GRAD_SUMSQ 43 /* MAX: largest whole-buffer sum of g^2 of one call */
#define RLCA_PPO_DIAG_COLUMNS 44

/* One minibatch into the row acc_dev.  Inputs as rlca_ppo_loss_fwd_bwd_weighted gets them after the same
 * rlca_policy_forward; new_lp and r are that kernel's own fp32 arithmetic, bit for bit (one device function).
 * action_bound = {lo0, lo1, hi0, hi1}, a HOST array.  Per-row terms are fp32, sums float64; one CTA with a fixed
 * reduction tree and one thread per column adding into acc_dev in stream order, no atomics: the same input gives the
 * same bits.  1 <= nb <= max_batch of `pol`; a NULL pointer or another nb is RLCA_ERR_INVALID. */
int rlca_ppo_diag_accumulate(rlca_policy *pol, const float *params_dev, const float *value_dev,
                             const float *mean_dev, const float *action_dev, const float *old_logprob_dev,
                             const float *adv_dev, const float *target_dev, int32_t nb, float clip_value,
                             const float *action_bound, double *acc_dev, void *stream);

/* Sum of g^2 of every tensor of the flat gradient buffer (the padding between tensors is not read) into the
 * RLCA_PPO_DIAG_GRAD_* columns of the row acc_dev: the per-tensor sums are added, the whole-buffer sum is merged into
 * the max column, and the step count goes up by one.  Two launches, fixed chunks and a fixed order of the partial sums
 * in float64 (scratch in `pol`), no atomics.  Call it after rlca_policy_backward on the same stream and BEFORE the
 * gradient exchange and the optimizer step: it measures the LOCAL gradient as the backward wrote it - scaled by
 * grad_weight, and under data parallelism this rank's share of the step's gradient, not the all-reduced one. */
int rlca_grad_sumsq(rlca_policy *pol, const float *grads_dev, double *acc_dev, void *stream);

/* Behaviour-cloning loss of one minibatch and its gradient w.r.t. the network outputs (the SL-policy, DESIGN.md §9g):
 * loss = mean over rows of sum_k (mean_k - target_k)^2, target_action_dev (nb,2) the demonstrated action.
 * losses_dev[0] = loss.  The output gradients stay in the workspace for rlca_policy_backward: the value's is 0, so the
 * critic tower's gradients are exactly 0, and so is the logstd gradient. */
int rlca_bc_loss_fwd_bwd(rlca_policy *pol, const float *params_dev, const float *mean_dev, const float *target_action_dev,
                         int32_t nb, float *losses_dev, void *stream);

/* Backward of the whole network for the batch of the last rlca_policy_forward: writes the
 * flat gradient buffer (RLCA_POLICY_NPARAMS floats; overwritten, not accumulated).
 * Stream semantics: the call orders all of its work after what is already enqueued on `stream`, and everything the
 * caller enqueues on `stream` afterwards (all-reduce, optimizer, the next forward) after all of its work - as if it had
 * run on `stream` alone.  Internally the weight / bias gradients and the operand transposes that are not on the chain
 * heads -> dX -> dF -> conv towers run on two streams owned by the workspace (forked and joined with events; no host
 * synchronisation).  RLCA_BWD_STREAMS=0 in the environment when the workspace is created keeps one stream;
 * so does a gradient event (rlca_policy_set_grad_event). */
int rlca_policy_backward(rlca_policy *pol, const float *params_dev, const float *obs_dev, const float *gs_dev,
                         int32_t nb, float *grads_dev, void *stream);

/* torch.optim.Adam step (ppo_stage1.py:179: lr 5e-5, betas (0.9,0.999), eps 1e-8, no decay),
 * bias-corrected, step counted from 1, over n contiguous floats. */
int rlca_adam_step(float *params_dev, const float *grads_dev, float *exp_avg_dev, float *exp_avg_sq_dev, int64_t n,
                   float lr, float beta1, float beta2, float eps, int32_t step, float grad_scale, void *stream);

/* The same step for the flat parameter buffer of a policy whose workspace is `pol` (all RLCA_POLICY_NTENSORS tensors,
 * padded layout of rlca_policy_param_offset): one kernel that also writes the derived copies of the fc1 weights the
 * tensor-core GEMMs read (tf32 hi / lo parts and their transposes), so the next rlca_policy_forward does not spend a
 * pass on them.  Same arithmetic, bit for bit, as rlca_adam_step followed by rlca_policy_weights_changed. */
int rlca_policy_adam_step(rlca_policy *pol, float *params_dev, const float *grads_dev, float *exp_avg_dev,
                          float *exp_avg_sq_dev, float lr, float beta1, float beta2, float eps, int32_t step,
                          float grad_scale, void *stream);

/* generate_train_data (model/ppo.py:122-139): GAE(gamma, lam) over (T,N) time-major arrays,
 * reverse recurrence evaluated in float64 like the reference's numpy; fp32 outputs. */
int rlca_gae(const float *rewards_dev, const float *values_dev, const float *last_value_dev, const uint8_t *dones_dev,
             int32_t num_step, int32_t num_env, float gamma, float lam, float *targets_dev, float *advs_dev,
             void *stream);

/* advs = (advs - mean)/std over the whole rollout (model/ppo.py:148: numpy mean/std, ddof 0, float64, no epsilon)
 * in two phases so that a data-parallel caller can all-reduce moments_dev (3 doubles: sum, sum of squares,
 * count) in between. */
int rlca_adv_moments(const float *x_dev, int64_t n, double *moments_dev, void *stream);
int rlca_adv_apply(const float *x_dev, int64_t n, const double *moments_dev, float *out_dev, void *stream);

/* dst[i,:] = src[idx[i],:] (rows of row_floats floats): random minibatch assembly (model/ppo.py:158-169). */
int rlca_gather_rows(const float *src_dev, const int64_t *idx_dev, int32_t row_floats, int32_t nrows, float *dst_dev,
                     void *stream);

/* The same for all arrays of a minibatch in ONE launch (the reference indexes obs, goal, speed, action, logprob, adv,
 * target with the same sampler index, model/ppo.py:162-169): dst[a][i,:] = src[a][idx[i],:], rows of row_floats[a]
 * floats, a < narrays <= RLCA_GATHER_MAX.  src / dst / row_floats are HOST arrays of device pointers / sizes. */
#define RLCA_GATHER_MAX 8
int rlca_gather_minibatch(const float *const *src_dev, const int32_t *row_floats, int32_t narrays,
                          const int64_t *idx_dev, int32_t nrows, float *const *dst_dev, void *stream);

/* Observation stack push (the deque of ppo_stage1.py:60,87-89): stack_out[:,0:2] = stack_in[:,1:3],
 * stack_out[:,2] = obs; agents whose flags say was_reset get three copies of obs. */
int rlca_obs_stack_push(const float *stack_in_dev, const float *obs_dev, const uint8_t *flags_dev, int32_t n,
                        int32_t beams, float *stack_out_dev, void *stream);

/* =====================================================================================
 * Evaluation (csrc/rlca_eval.cu, DESIGN.md §9c): per-episode records and the metrics of the paper this reference
 * accompanies - success rate, extra time, extra distance, average speed.
 * ===================================================================================== */

/* Per-agent tracking state, N = robots_per_world * num_worlds rows; the caller zeroes path / count / open and sets
 * closed to -1 before the first tick it tracks.
 *   path     length of the running episode's path so far, metres
 *   count    episodes that ended so far; only the first `episodes` of them are recorded
 *   closed   episode index (state meta.y) of the last ended episode, -1 = none: nothing is tracked until the agent
 *            starts a new episode (auto_reset 0: the caller resets it; 2: its group re-spawns)
 *   open     1 = the agent is in an episode that has not ended (written by every rlca_eval_track)
 *   records  (N, episodes, 4) result code (1 Reach Goal, 2 Crashed, 3 Time out), ticks, path length, straight-line
 *            start -> goal distance (init and goal of the eplog row) */
typedef struct rlca_eval_state {
    double *path_dev;
    int32_t *count_dev;
    int32_t *closed_dev;
    int32_t *open_dev;
    float *records_dev;
    int32_t episodes;
} rlca_eval_state;

/* One launch after each rlca_env_step, with the same cfg, state buffers and io: reads the action, flags, eplog, the
 * poses of state_in / state_out and the episode indices, and appends a record for every agent whose episode ended. */
int rlca_eval_track(const rlca_env_config *cfg, const rlca_env_state *state_in, const rlca_env_state *state_out,
                    const rlca_step_io *io, const rlca_eval_state *ev, void *stream);

/* Per-world float64 partials of the records of worlds [world_begin, world_begin + world_count) of the shard, in a
 * fixed order without atomics: partials_dev (world_count, RLCA_EVAL_NPARTIALS).  With T = ticks * dt and
 * L = max(distance - goal_radius, 0), over the episodes that reached the goal: travel time T, extra time T - L / v_max,
 * extra distance path - L, average speed path / T.  Totals are the partials summed in global world order. */
#define RLCA_EVAL_REACHED 0          /* episodes with result 1 */
#define RLCA_EVAL_CRASHED 1          /* result 2 */
#define RLCA_EVAL_TIMED_OUT 2        /* result 3 */
#define RLCA_EVAL_UNFINISHED 3       /* agents with fewer than `episodes` records that are in an episode */
#define RLCA_EVAL_SUM_TIME 4         /* sum, sum of squares of travel time (4, 5), extra time (6, 7), */
                                     /*   extra distance (8, 9), average speed (10, 11) */
#define RLCA_EVAL_SUM_STRAIGHT 12    /* sum of the straight-line start -> goal distance */
#define RLCA_EVAL_SUM_PATH 13        /* sum of the path length */
#define RLCA_EVAL_NPARTIALS 14
int rlca_eval_reduce(const rlca_env_config *cfg, const rlca_eval_state *ev, int32_t world_begin, int32_t world_count,
                     double *partials_dev, void *stream);
/* The same reduction from HOST buffers (no device needed; the code rlca_eval_reduce runs). */
int rlca_eval_reduce_host(const rlca_env_config *cfg, const float *records_host, const int32_t *count_host,
                          const int32_t *open_host, int32_t episodes, int32_t world_begin, int32_t world_count,
                          double *partials_host);
/* The same partials split by an agent mask (N uint8, DESIGN.md §9h): partials_dev (world_count, 2,
 * RLCA_EVAL_NPARTIALS), row 0 over the agents with mask 0 and row 1 over the others, each in the order of
 * rlca_eval_reduce (one thread per world and row, no atomics).  A NULL mask is RLCA_ERR_INVALID. */
int rlca_eval_reduce_split(const rlca_env_config *cfg, const rlca_eval_state *ev, const uint8_t *mask_dev,
                           int32_t world_begin, int32_t world_count, double *partials_dev, void *stream);
int rlca_eval_reduce_split_host(const rlca_env_config *cfg, const float *records_host, const int32_t *count_host,
                                const int32_t *open_host, const uint8_t *mask_host, int32_t episodes,
                                int32_t world_begin, int32_t world_count, double *partials_host);

/* =====================================================================================
 * ORCA-DD baseline controller (csrc/rlca_orca.cu, DESIGN.md §9d): reciprocal velocity obstacles (van den Berg et al.
 * 2011) over the robots of each world with a differential-drive heading tracker.  Not NH-ORCA; static map ignored.
 * ===================================================================================== */

/* One action per agent from the state the next rlca_env_step reads (pose, goal, meta of `state`): position, heading,
 * goal, and the current velocity goal.z * (cos, sin)(theta), 0 when the stall flag meta.z is set.  Neighbours are the
 * other robots of the same world closer than neighbour_dist; radius is one robot's (the pair's is 2 * radius),
 * time_horizon is tau in s, heading_gain k_w in 1/s.
 *   action_dev    (N,2) raw action (v, w) for rlca_env_step
 *   velocity_dev  optional (N,2) ORCA velocity in the world frame
 *   status_dev    optional (N) 0 = LP feasible, 1 = least-penetration fallback
 * Every parameter must be finite and > 0 (RLCA_ERR_INVALID otherwise). */
int rlca_orca_action(const rlca_env_config *cfg, const rlca_env_state *state, float radius, float neighbour_dist,
                     float time_horizon, float heading_gain, float *action_dev, float *velocity_dev,
                     int32_t *status_dev, void *stream);
/* The same from HOST buffers (pose, goal: (N,4) float; meta: (N,4) int32), by serial loops over the same per-line code;
 * the outputs equal rlca_orca_action's bit for bit.  velocity_host and status_host may be NULL. */
int rlca_orca_action_host(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                          const int32_t *meta_host, float radius, float neighbour_dist, float time_horizon,
                          float heading_gain, float *action_host, float *velocity_host, int32_t *status_host);

/* Non-cooperative robots (DESIGN.md §9h): drive straight to the goal and ignore every other robot and the map.
 * action_dev (N,2) is read and written in place: for every agent with mask_dev[a] != 0 (N uint8) the row becomes
 * ORCA-DD's action for an agent without neighbours, with v_max = speed and k_w = heading_gain (w bounds from cfg);
 * rows with mask 0 are not touched.  speed must be finite and in (0, cfg->v_max], heading_gain finite and > 0, and
 * no buffer may be NULL (RLCA_ERR_INVALID otherwise). */
int rlca_noncoop_action(const rlca_env_config *cfg, const rlca_env_state *state, const uint8_t *mask_dev, float speed,
                        float heading_gain, float *action_dev, void *stream);
/* The same from HOST buffers (pose, goal: (N,4) float; meta: (N,4) int32); equal to rlca_noncoop_action bit for bit. */
int rlca_noncoop_action_host(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                             const int32_t *meta_host, const uint8_t *mask_host, float speed, float heading_gain,
                             float *action_host);

/* Social-force crowd (DESIGN.md §9t): masked agents driven by a Helbing-Molnar style social force that avoid each
 * other, the static map and (see_robots != 0) the other agents.  action_dev (N,2) is read and written in place: for
 * every agent i with mask_dev[i] != 0 (N uint8), from the state the next rlca_env_step reads, in float32:
 *   p, heading (c, s), v = last command along the heading (0 when the stall flag is set);
 *   u0 = the non-cooperative driver's preferred velocity at v_max = speed;  f = (u0 - v) (1 / relax_time);
 *   for every other agent j of the world with 0 < d = |p_i - p_j| < neighbour_dist (see_robots == 0: mask[j] != 0
 *   only), n = (p_i - p_j) / d, t = n rotated by +90 degrees, cos phi = -n . (c, s),
 *   w = anisotropy + (1 - anisotropy)(1 + cos phi) / 2:  f += strength exp((2 radius - d) / range) w (n + side_bias t);
 *   with an obstacle set, for every segment of the agent's bin list within wall_dist with the agent strictly on its
 *   free side, q its nearest point, d = |p - q| > 0, n = (p - q) / d:
 *   f += wall_strength exp((radius - d) / wall_range) n;
 *   u = v + f cfg.dt on the disk of radius speed; the action is ORCA-DD's heading tracker on u with k_w = heading_gain
 *   (w bounds from cfg).
 * Rows with mask 0 are not touched; obstacles NULL is map-blind.  RLCA_ERR_INVALID for a NULL buffer, speed outside
 * (0, cfg->v_max], relax_time, range, wall_range, radius, neighbour_dist or heading_gain not finite and > 0, strength
 * or wall_strength not finite and >= 0, anisotropy outside [0, 1], side_bias not finite and >= 0, wall_dist not finite
 * and > 0 or above the obstacle set's max_range. */
typedef struct rlca_crowd_params {
    float speed, relax_time, strength, range, anisotropy, side_bias, radius, neighbour_dist;
    float wall_strength, wall_range, wall_dist, heading_gain;
    int32_t see_robots;
} rlca_crowd_params;
int rlca_crowd_action(const rlca_env_config *cfg, const rlca_crowd_params *params, const rlca_env_state *state,
                      const uint8_t *mask_dev, struct rlca_orca_obstacles *obstacles, float *action_dev, void *stream);
/* The same from HOST buffers (pose, goal: (N,4) float; meta: (N,4) int32); equal to rlca_crowd_action bit for bit. */
int rlca_crowd_action_host(const rlca_env_config *cfg, const rlca_crowd_params *params,
                           struct rlca_orca_obstacles *obstacles, const float *pose_host, const float *goal_host,
                           const int32_t *meta_host, const uint8_t *mask_host, float *action_host);
/* The kernel's e^x (a cephes-style polynomial that rounds alike on host and device) on n host floats, for tests. */
int rlca_crowd_expf_host(const float *x_host, int32_t n, float *out_host);

/* Hybrid controller (DESIGN.md §9j): switches a policy's action per agent by the nearest return of its newest scan.
 * With m the minimum of frame 2 of the (N,3,beams) scan stack the tick reads (values scan / range_max - 0.5) and
 * d = (m + 0.5f) * cfg->range_max in metres, action_dev (N,2) is rewritten in place:
 *   mode 1  d > r_safe   the non-cooperative driver's action at speed cfg->v_max with k_w = heading_gain
 *   mode 2  d < r_risk   (fminf(v, v_safe), w)
 *   mode 0  otherwise    unchanged
 * mode_dev (N uint8) receives the mode.  With open_dev (N int32, rlca_eval_state.open) and counts_dev (N,3 int32) both
 * set, counts[a][mode] += 1 for every agent with open[a] != 0; both NULL counts nothing.  Needs
 * 0 <= r_risk <= r_safe <= cfg->range_max (all finite), v_safe in (0, cfg->v_max], heading_gain finite and > 0, and
 * no NULL buffer (RLCA_ERR_INVALID otherwise).  r_risk = 0 turns mode 2 off; r_safe = range_max turns mode 1 off. */
typedef struct rlca_hybrid_params {
    float r_safe;
    float r_risk;
    float v_safe;
    float heading_gain;
} rlca_hybrid_params;
int rlca_hybrid_action(const rlca_env_config *cfg, const rlca_hybrid_params *params, const rlca_env_state *state,
                       const float *stack_dev, const int32_t *open_dev, float *action_dev, uint8_t *mode_dev,
                       int32_t *counts_dev, void *stream);
/* The same from HOST buffers (stack (N,3,beams) float; pose, goal: (N,4) float; meta: (N,4) int32); equal to
 * rlca_hybrid_action bit for bit. */
int rlca_hybrid_action_host(const rlca_env_config *cfg, const rlca_hybrid_params *params, const float *stack_host,
                            const float *pose_host, const float *goal_host, const int32_t *meta_host,
                            const int32_t *open_host, float *action_host, uint8_t *mode_host, int32_t *counts_host);

/* =====================================================================================
 * NH-ORCA baseline controller (csrc/rlca_orca.cu, DESIGN.md §9e): ORCA for non-holonomic robots (Alonso-Mora,
 * Breitenmoser, Rufli, Beardsley, Siegwart, DARS 2010), the paper's baseline.  Static map ignored.
 *
 * Tracking: a holonomic velocity at speed V and angle th in (-pi, pi] from the heading is tracked by turning at
 * w = th / T_th, T_th = max(T, th / w_max) (th < 0: th / w_min), T = heading_time, while driving at
 * v* = V (th/2) cot(th/2) (V at th = 0), then straight at V.  Its largest distance from V t (cos th, sin th) is
 * V T_th |sin(th/2)|.  The robot may choose among the velocities of P, a convex polygon of at most
 * RLCA_NH_ORCA_VERTS vertices that contains the origin strictly and lies inside S_E = {V <= min(v_max, E / (T_th
 * |sin(th/2)|))}, E = tracking_error; P is built on the host in float64 from (E, T, v_max, w_min, w_max).
 * ORCA: the neighbours, half-planes and preferred velocity of rlca_orca_action with the pair's radius
 * 2 * (radius + tracking_error).  The LP's lines are P's edges (rotated by the heading) first, then the ORCA lines;
 * its optimum is the velocity nearest to the preferred one (status 0).  If an ORCA line makes it infeasible, the
 * least-penetration program takes over from that line with P's edges kept hard (status 1).
 * Action: (v*, th / T_th) of the chosen velocity clipped to the action bounds; (0, 0) for a speed <= 1e-6.
 * Every parameter must be finite and > 0, and cfg must have v_min <= 0 < v_max and w_min < 0 < w_max
 * (RLCA_ERR_INVALID otherwise).
 * ===================================================================================== */
#define RLCA_NH_ORCA_VERTS 32
/*   action_dev    (N,2) raw action (v, w) for rlca_env_step
 *   velocity_dev  optional (N,2) chosen holonomic velocity in the world frame
 *   status_dev    optional (N) 0 = LP feasible, 1 = least-penetration fallback */
int rlca_nh_orca_action(const rlca_env_config *cfg, const rlca_env_state *state, float radius, float neighbour_dist,
                        float time_horizon, float tracking_error, float heading_time, float *action_dev,
                        float *velocity_dev, int32_t *status_dev, void *stream);
/* The same from HOST buffers, by serial loops over the same per-line code; the outputs equal rlca_nh_orca_action's
 * bit for bit.  velocity_host and status_host may be NULL. */
int rlca_nh_orca_action_host(const rlca_env_config *cfg, const float *pose_host, const float *goal_host,
                             const int32_t *meta_host, float radius, float neighbour_dist, float time_horizon,
                             float tracking_error, float heading_time, float *action_host, float *velocity_host,
                             int32_t *status_host);
/* P in the robot frame (x along the heading): *nverts vertices, counter-clockwise, into verts_host
 * (room for RLCA_NH_ORCA_VERTS x 2 floats). */
int rlca_nh_orca_polygon_host(const rlca_env_config *cfg, float tracking_error, float heading_time, int32_t *nverts,
                              float *verts_host);

/* =====================================================================================
 * Static obstacles for both ORCA controllers (csrc/rlca_orca.cu, DESIGN.md §9f): the obstacle half-planes of RVO2
 * (van den Berg et al. 2011, §6) from the boundary of the static grid.
 *
 * Obstacle region: the union of the squares of the non-zero cells (cell (i, j) covers x in [(i - origin_cx) res,
 * (i + 1 - origin_cx) res), likewise y); cells outside the grid are free.  Its boundary is a set of closed loops of
 * segments, occupied cells on the LEFT of every segment (counter-clockwise round obstacles, clockwise round holes),
 * each a maximal run of collinear cell edges; two occupied cells that touch only at a corner are connected (no loop
 * passes between them).  A vertex is convex when the loop turns left there.  Built on the host in float64 and rounded
 * to float once; no device is needed.  The lookup bins are RLCA_ORCA_MAP_BIN m squares; each lists the segments within
 * max_range of it, at most RLCA_ORCA_MAP_MAX_CANDIDATES (RLCA_ERR_UNSUPPORTED otherwise, never truncated).  The device
 * copy is made at creation when a device is present, else on first device use, on the current device; a set serves
 * that one device.
 *
 * The _map entries take the obstacle set and obstacle_time_horizon tau_o next to the controller's parameters.  The
 * obstacle radius r_o is the controller's own (ORCA-DD: radius; NH-ORCA: radius + tracking_error), and
 * tau_o * v_max + r_o must not exceed max_range (RLCA_ERR_INVALID).  Per agent (position and current velocity as the
 * map-blind controllers take them): the candidates are the segments closer than tau_o * v_max + r_o with the agent
 * strictly on their free side, taken in order of (squared distance in float32, segment index); a segment whose two
 * vertices, scaled by 1 / tau_o, lie at least r_o / tau_o beyond an obstacle line built so far is skipped, otherwise it
 * adds RVO2's obstacle line (none for a colliding non-convex vertex or a nearest point on a foreign leg).  At most
 * RLCA_ORCA_MAP_MAX_LINES obstacle lines are kept, the nearest; the LP's lines are [P's edges (NH-ORCA)], the obstacle
 * lines, the agent lines, and P's edges and the obstacle lines are hard in the least-penetration fallback.
 *   status  bit 0: the least-penetration fallback ran; bit 1: it started at an obstacle line (rounding made the hard
 *           lines infeasible; the velocity may then violate obstacle lines); bit 2: obstacle lines were dropped at
 *           RLCA_ORCA_MAP_MAX_LINES.
 * With an all-free grid the outputs equal the map-blind entries' bit for bit.
 * ===================================================================================== */
#define RLCA_ORCA_MAP_BIN 0.25f
#define RLCA_ORCA_MAP_MAX_CANDIDATES 512
#define RLCA_ORCA_MAP_MAX_LINES 64
typedef struct rlca_orca_obstacles rlca_orca_obstacles;
/* cells_host: grid_h * grid_w bytes, row-major, 0 = free (rlca_env_set_map's layout); cfg gives resolution and
 * origin_cx / origin_cy; max_range in m, finite and > 0. */
int rlca_orca_obstacles_create(const rlca_env_config *cfg, const uint8_t *cells_host, int32_t grid_w, int32_t grid_h,
                               float max_range, rlca_orca_obstacles **out);
int rlca_orca_obstacles_destroy(rlca_orca_obstacles *obs);
/* The segments: *nsegments; optional *max_list (longest bin list); optional points_host [4 * nsegments] float
 * (x0, y0, x1, y1) and links_host [3 * nsegments] int32 (previous segment, next segment, convex flag of the start
 * vertex).  Segments of one loop are consecutive. */
int rlca_orca_obstacles_segments(const rlca_orca_obstacles *obs, int32_t *nsegments, int32_t *max_list,
                                 float *points_host, int32_t *links_host);
int rlca_orca_action_map(const rlca_env_config *cfg, const rlca_env_state *state, rlca_orca_obstacles *obstacles,
                         float radius, float neighbour_dist, float time_horizon, float heading_gain,
                         float obstacle_time_horizon, float *action_dev, float *velocity_dev, int32_t *status_dev,
                         void *stream);
int rlca_orca_action_map_host(const rlca_env_config *cfg, rlca_orca_obstacles *obstacles, const float *pose_host,
                              const float *goal_host, const int32_t *meta_host, float radius, float neighbour_dist,
                              float time_horizon, float heading_gain, float obstacle_time_horizon, float *action_host,
                              float *velocity_host, int32_t *status_host);
int rlca_nh_orca_action_map(const rlca_env_config *cfg, const rlca_env_state *state, rlca_orca_obstacles *obstacles,
                            float radius, float neighbour_dist, float time_horizon, float tracking_error,
                            float heading_time, float obstacle_time_horizon, float *action_dev, float *velocity_dev,
                            int32_t *status_dev, void *stream);
int rlca_nh_orca_action_map_host(const rlca_env_config *cfg, rlca_orca_obstacles *obstacles, const float *pose_host,
                                 const float *goal_host, const int32_t *meta_host, float radius, float neighbour_dist,
                                 float time_horizon, float tracking_error, float heading_time,
                                 float obstacle_time_horizon, float *action_host, float *velocity_host,
                                 int32_t *status_host);
/* The obstacle lines of one agent as the _map entries build them, for tests: *nlines lines (point x, y, unit
 * direction x, y; allowed side on the left) into lines_host [4 * RLCA_ORCA_MAP_MAX_LINES], *dropped as status bit 2. */
int rlca_orca_obstacle_lines_host(const rlca_env_config *cfg, rlca_orca_obstacles *obstacles, const float *pose_host,
                                  const float *goal_host, const int32_t *meta_host, int32_t agent,
                                  float obstacle_radius, float obstacle_time_horizon, int32_t *nlines,
                                  int32_t *dropped, float *lines_host);

/* =====================================================================================
 * Demonstration recording (csrc/rlca_demo.cu, DESIGN.md §9g): (observation, expert action) pairs for supervised
 * training of the policy, appended on the device while a controller drives the env.
 * ===================================================================================== */

/* A fixed-capacity dataset of rows, in device memory the caller owns:
 *   obs     (capacity, 3 * beams) the scan stack the controller's tick reads (stack_in of rlca_env_step)
 *   gs      (capacity, 4) local goal x, y + speed v, w before the tick
 *   action  (capacity, 2) the action clipped to [v_min, v_max] x [w_min, w_max] as the tick clips it (non-finite -> 0)
 *   count   2 int64: [0] rows held, [1] zero between calls (completion ticket).  The caller zeroes both. */
typedef struct rlca_demo_set {
    float *obs_dev;
    float *gs_dev;
    float *action_dev;
    int64_t *count_dev;
    int64_t capacity;
} rlca_demo_set;

/* One launch before the rlca_env_step it records, with that tick's cfg, state_in and io: reads io->stack_in_dev,
 * io->gs_dev, io->action_dev, state->meta_dev (auto_reset 2) and io->flags_dev as the PREVIOUS tick's flags (auto_reset
 * 0; NULL = no agent was done).  An agent is recorded when its action drives an episode that has not ended:
 * auto_reset 1 always, auto_reset 2 when not latched (meta.w == 0), auto_reset 0 when not done on the previous tick.
 * Rows are appended in agent order; a full dataset keeps its first `capacity` rows.  No host synchronisation.
 * io->live_dev must be NULL (RLCA_ERR_UNSUPPORTED); 3 * beams must be a multiple of 4; obs and gs buffers 16-byte,
 * action and count 8-byte aligned. */
int rlca_demo_append(const rlca_env_config *cfg, const rlca_env_state *state, const rlca_step_io *io,
                     const rlca_demo_set *demo, void *stream);

/* =====================================================================================
 * Random layouts (csrc/rlca_layout.cu, DESIGN.md §9i): every world of an evaluation gets its own starts and goals,
 * drawn on the device once before the episode.
 * ===================================================================================== */

/* side        edge of the square [-side/2, side/2]^2 that holds every start and goal, m
 * separation  least distance between two starts and between two goals, m
 * min_travel  least distance from a robot's start to its goal, m */
typedef struct rlca_layout_params {
    float side;
    float separation;
    float min_travel;
} rlca_layout_params;

/* Writes a layout into `state` in place.  World w (global index cfg->world_offset + w), robots r = 0 .. R-1 in order:
 * the start is the first try k < cfg->max_reject whose uniform draw in the square is at least `separation` from the
 * starts of robots 0 .. r-1; the goal the first try whose draw is at least `min_travel` from this start and
 * `separation` from the goals of robots 0 .. r-1; the heading one draw u * 2 pi wrapped into (-pi, pi].  Draws are the
 * env's Philox draws with agent = global world * R + r, episode 0, draw k and purposes 3 (start), 4 (goal), 5
 * (heading), so a world's layout does not depend on num_worlds or on sharding.  Distances are compared squared in
 * float32.  Written per robot: pose = (x, y, theta, pre_distance) with pre_distance 0 when cfg->pre_distance_zero and
 * |goal - start| otherwise, goal.xy, acc.zw = (x, y) (the init pose); every other field is kept.
 *   status_dev  (num_worlds) int32: 0 = placed; 1 + r when robot r found no accepted try, and the world's rows are then
 *               left untouched
 * RLCA_ERR_INVALID for a NULL pointer, robots_per_world outside 2..64, side not finite and > 0, min_travel outside
 * [0, side sqrt(2)], or separation <= 2 (r_c + sqrt(2) resolution), r_c = sqrt(half_len^2 + half_wid^2): two
 * footprints that far apart share no cell whatever their headings. */
int rlca_layout_random(const rlca_env_config *cfg, const rlca_layout_params *params, const rlca_env_state *state,
                       int32_t *status_dev, void *stream);
/* The same from HOST buffers (pose, goal, acc: (N,4) float; status: (num_worlds) int32) by a sequential loop over
 * the tries; the outputs equal rlca_layout_random's bit for bit. */
int rlca_layout_random_host(const rlca_env_config *cfg, const rlca_layout_params *params, float *pose_host,
                            float *goal_host, float *acc_host, int32_t *status_host);

/* Training on random layouts (DESIGN.md §9k): one launch after each rlca_env_step of an env with auto_reset 0, in place
 * on the state that tick wrote, with that tick's flags.  Per world (global index cfg->world_offset + w):
 *   - a latched robot (meta.w != 0) is parked: goal.zw (its last command) = 0 and live[a] = 0; every other robot gets
 *     live[a] = 1.  Passed as the next tick's io->live_dev, a parked robot stands still.
 *   - a world whose robots are all latched is re-laid at once: the draws of rlca_layout_random with episode
 *     e = meta.y + 1 of robot 0 instead of 0, written as the tick's re-spawn writes a new episode (pose, goal.xy,
 *     pre_distance, acc.zw = start, acc.x = 0, meta.x = 1, meta.y = e, meta.w = 0, stall flag and acc.y kept) with
 *     goal.zw = 0, live = 1 and flags[a].w (was_reset) = 1.
 *   - status_dev[w] = 0, or 1 + r when a re-layout could not place robot r; that world keeps its rows, parked.
 * RLCA_ERR_INVALID for what rlca_layout_random rejects, cfg->auto_reset != 0, or a NULL buffer (meta included).
 *   flags_dev (N) uchar4, live_dev (N) uint8, status_dev (num_worlds) int32. */
int rlca_layout_respawn(const rlca_env_config *cfg, const rlca_layout_params *params, const rlca_env_state *state,
                        uint8_t *flags_dev, uint8_t *live_dev, int32_t *status_dev, void *stream);
/* The same from HOST buffers (pose, goal, acc (N,4) float; meta (N,4) int32; flags (N,4) uint8; live (N) uint8;
 * status (num_worlds) int32) by the sequential loop of rlca_layout_random_host; the outputs equal the device's bit for
 * bit. */
int rlca_layout_respawn_host(const rlca_env_config *cfg, const rlca_layout_params *params, float *pose_host,
                             float *goal_host, float *acc_host, int32_t *meta_host, uint8_t *flags_host,
                             uint8_t *live_host, int32_t *status_host);
/* For every agent with flags_dev[a].w set: stack_dev[a][0..2] = obs_dev[a] (three copies of the scan, (N,3,beams)
 * float) and gs_dev[a] = gs_src_dev[a] ((N,4) float); every other row is untouched.  Run after rlca_env_observe on
 * the state rlca_layout_respawn re-laid, so a re-laid agent's FIFO and goal | speed are those the tick writes after
 * an in-tick re-spawn.  RLCA_ERR_INVALID for a NULL pointer, 3 * beams not a multiple of 4, or a buffer that is not
 * 16-byte aligned. */
int rlca_stack_refresh(const rlca_env_config *cfg, const uint8_t *flags_dev, const float *obs_dev,
                       const float *gs_src_dev, float *stack_dev, float *gs_dev, void *stream);

/* =====================================================================================
 * Arena layouts (csrc/rlca_layout.cu, DESIGN.md §9v): one map holds T walled arenas with their own obstacles
 * (rl_collision_avoidance_b200/arenas.py), and every world lays its robots out in one arena's placeable cells.
 * ===================================================================================== */

/* The placeable cells of T arenas: arena a owns cells[cell_off[a] .. cell_off[a + 1]), each packed cx | cy << 16
 * (map column and row).  Device pointers for the device entries, host pointers for the host twins. */
typedef struct rlca_arena_tables {
    int32_t num_arenas;          /* T >= 1 */
    const int32_t *cell_off;     /* T + 1 offsets: cell_off[0] = 0, strictly increasing */
    const int32_t *cells;        /* cell_off[T] packed cells, each on the cfg's grid_w x grid_h map */
} rlca_arena_tables;

/* RLCA_OK when host tables hold what the device entries rely on: cell_off[0] = 0, no empty arena, increasing
 * offsets, every cell on the map.  The device entries cannot read the tables without a synchronisation; run this on
 * the host copy before uploading them. */
int rlca_arena_tables_check(const rlca_env_config *cfg, const rlca_arena_tables *tables_host);

/* rlca_layout_random's layout in arenas.  World w (global index g = cfg->world_offset + w) lays out in arena
 *   pick 0: g mod T;  pick 1: (m T) >> 24, m = 2^24 u0 of the draw (agent g R, episode, draw 0, purpose 0xA0),
 * and try k of robot r's start (goal) draws (agent g R + r, episode, draw k, purpose 0xA3 (0xA4)): the cell
 * cells[cell_off[a] + ((m n_a) >> 24)], m = 2^24 u0, n_a the arena's cell count, and the point
 * x = ((cx - origin_cx) + u1) res, y = ((cy - origin_cy) + u2) res in float32.  Acceptance (separation, min_travel),
 * heading (purpose 5), the records written and status_dev are rlca_layout_random's; params->side is not read.
 * RLCA_ERR_INVALID for what rlca_layout_random rejects other than side, min_travel not finite and >= 0, NULL tables,
 * T < 1 or pick outside {0, 1}. */
int rlca_layout_arena(const rlca_env_config *cfg, const rlca_layout_params *params, const rlca_arena_tables *tables,
                      int32_t pick, const rlca_env_state *state, int32_t *status_dev, void *stream);
/* The same from HOST buffers and host tables by the sequential loop; equal to the device's bit for bit.  Also
 * RLCA_ERR_INVALID for what rlca_arena_tables_check rejects. */
int rlca_layout_arena_host(const rlca_env_config *cfg, const rlca_layout_params *params,
                           const rlca_arena_tables *tables_host, int32_t pick, float *pose_host, float *goal_host,
                           float *acc_host, int32_t *status_host);
/* rlca_layout_respawn with the arena sampler: park the latched robots, re-lay a world whose robots are all latched
 * at episode e = meta.y + 1 (pick 1 draws its arena at that episode too).  rlca_stack_refresh follows as for
 * rlca_layout_respawn.  RLCA_ERR_INVALID for what rlca_layout_arena rejects, cfg->auto_reset != 0 or a NULL buffer. */
int rlca_layout_arena_respawn(const rlca_env_config *cfg, const rlca_layout_params *params,
                              const rlca_arena_tables *tables, int32_t pick, const rlca_env_state *state,
                              uint8_t *flags_dev, uint8_t *live_dev, int32_t *status_dev, void *stream);
int rlca_layout_arena_respawn_host(const rlca_env_config *cfg, const rlca_layout_params *params,
                                   const rlca_arena_tables *tables_host, int32_t pick, float *pose_host,
                                   float *goal_host, float *acc_host, int32_t *meta_host, uint8_t *flags_host,
                                   uint8_t *live_host, int32_t *status_host);

/* =====================================================================================
 * Safety metrics (csrc/rlca_safety.cu, DESIGN.md §9m): how closely robots pass and why they crash, per episode of the
 * evaluation tracker above.
 *
 * Footprint: the rectangle of half extents cfg->half_len, cfg->half_wid at the robot's pose (the tick's corners).
 * Separation of a robot at a tick: the least distance between its footprint and the footprint of any other robot of
 * its world, 0 when two intersect, +inf in a world of one robot; the partner is the robot that attains it (lowest
 * index on ties).  Every other robot of the world counts, finished or not: the tick's collision test sees them all.
 * Clearance of a robot at a tick: the nearest return of the scan the tick wrote, (min obs + 0.5) * range_max metres.
 * Contact bound: sqrt(2) resolution + 2 dt (v_max + max(|w_min|, |w_max|) r_c), r_c = sqrt(half_len^2 + half_wid^2):
 * two robots whose footprints come to share a cell within one tick started it no farther apart than that.
 * ===================================================================================== */
typedef struct rlca_safety_params {
    float near_dist;             /* a tick whose separation is below this is a near-miss tick; finite, >= 0 */
} rlca_safety_params;

/* Per-agent state, N rows; before the first tick it tracks the caller sets min_sep, min_clear and last_clear to +inf,
 * near to 0 and partner to -1.
 *   min_sep, partner   running episode: least separation so far and the robot (index in its world) it was to
 *   min_clear          running episode: least clearance so far
 *   last_clear         clearance of the previous tick's scan, taken at the pose the next tick starts from
 *   near               running episode: near-miss ticks
 *   records            (N, episodes, 4), slot for slot the tracker's records: minimum separation, minimum clearance,
 *                      near-miss ticks, and an integer held exactly by the float:
 *                        bits 0-1   crash cause: 0 not a crash, 1 static map, 2 robot
 *                        bit  2     cause robot, and last_clear was below the contact bound too ("both in range")
 *                        bits 8-15  1 + the robot (index in its world) a cause-robot crash is charged to, else 0
 *                        bits 16-23 1 + the partner of the minimum separation, 0 = none */
typedef struct rlca_safety_state {
    float *min_sep_dev;
    float *min_clear_dev;
    float *last_clear_dev;
    int32_t *near_dev;
    int32_t *partner_dev;
    float *records_dev;
    int32_t episodes;
} rlca_safety_state;

/* One launch after each rlca_env_step and BEFORE that tick's rlca_eval_track, with the same cfg, state buffers and
 * io: reads the poses of state_in / state_out, the episode indices of state_in, io->flags_dev, io->obs_dev and the
 * tracker's closed / count (never written), so a tick belongs to the episode the tracker assigns it to and a record
 * goes into the slot the tracker fills next.  Per tracked robot the tick's separation is taken at the poses of
 * state_out; for a robot the tick re-spawned (flags.w: state_out is the next episode's pose) at the poses of state_in,
 * all robots', and its scan is not folded.  A tick that ends an episode writes the record and resets the running
 * state, as does a re-spawn.  An episode that ends with result 2 gets its cause from the separation d0 of the robot at
 * the poses of state_in: static when d0 exceeds the contact bound, otherwise robot, charged to the partner of d0.
 * RLCA_ERR_INVALID for a NULL pointer, robots_per_world outside 1..64, episodes < 1 or different from the tracker's,
 * near_dist not finite or < 0. */
int rlca_safety_track(const rlca_env_config *cfg, const rlca_safety_params *params, const rlca_env_state *state_in,
                      const rlca_env_state *state_out, const rlca_step_io *io, const rlca_eval_state *ev,
                      const rlca_safety_state *ss, void *stream);
/* The same from HOST buffers (pose (N,4) float; meta (N,4) int32; flags (N,4) uint8; obs (N,beams) float; the rest as
 * the device state) by serial loops over the same code; the outputs equal rlca_safety_track's bit for bit. */
int rlca_safety_track_host(const rlca_env_config *cfg, const rlca_safety_params *params, const float *pose_in_host,
                           const int32_t *meta_in_host, const float *pose_out_host, const uint8_t *flags_host,
                           const float *obs_host, const int32_t *closed_host, const int32_t *count_host,
                           int32_t episodes, float *min_sep_host, float *min_clear_host, float *last_clear_host,
                           int32_t *near_host, int32_t *partner_host, float *records_host);
/* Separation of the footprints at pose_a_host[i] and pose_b_host[i] ((n,4) float x, y, theta, _), i < n, and the
 * contact bound of cfg: the code the tracker runs, for tests and tools (no device needed). */
int rlca_safety_separation_host(const rlca_env_config *cfg, const float *pose_a_host, const float *pose_b_host,
                                int32_t n, float *separation_host);
int rlca_safety_contact_host(const rlca_env_config *cfg, float *contact);

/* Per-world float64 partials of the safety records of worlds [world_begin, world_begin + world_count), one thread per
 * world in agent-then-record order, no atomics: partials_dev (world_count, RLCA_SAFETY_NPARTIALS).  The tracker's
 * state gives the number of records per agent and each record's result code.  With role_mask_dev (N uint8) the
 * partials are split as rlca_eval_reduce_split splits its own, partials_dev (world_count, 2, RLCA_SAFETY_NPARTIALS):
 * row 0 over the agents with mask 0, row 1 over the others.  Every column but the last is a sum; totals add them in
 * global world order and take the minimum of the last. */
#define RLCA_SAFETY_CRASH_STATIC 0         /* crashes with cause static */
#define RLCA_SAFETY_CRASH_ROBOT 1          /* cause robot */
#define RLCA_SAFETY_CRASH_BOTH_IN_RANGE 2  /* cause robot with a scan return within the contact bound as well */
#define RLCA_SAFETY_CRASH_INTO_MASKED 3    /* cause robot, charged to a robot with role mask != 0 (0 without a mask) */
#define RLCA_SAFETY_REACHED 4              /* episodes that reached the goal; the columns up to 12 are over these */
#define RLCA_SAFETY_REACHED_SEPARATION 5   /* ... with a finite minimum separation */
#define RLCA_SAFETY_SUM_SEPARATION 6       /* sum, sum of squares (6, 7) of the finite minimum separations */
#define RLCA_SAFETY_REACHED_CLEARANCE 8    /* ... with a finite minimum clearance */
#define RLCA_SAFETY_SUM_CLEARANCE 9        /* sum, sum of squares (9, 10) of the finite minimum clearances */
#define RLCA_SAFETY_NEAR_EPISODES 11       /* ... with at least one near-miss tick */
#define RLCA_SAFETY_SUM_NEAR_TICKS 12      /* their near-miss ticks */
#define RLCA_SAFETY_MIN_SEPARATION 13      /* least minimum separation of all recorded episodes, +inf when none */
#define RLCA_SAFETY_NPARTIALS 14
int rlca_safety_reduce(const rlca_env_config *cfg, const rlca_safety_state *ss, const rlca_eval_state *ev,
                       const uint8_t *role_mask_dev, int32_t world_begin, int32_t world_count, double *partials_dev,
                       void *stream);
/* The same reduction from HOST buffers (no device needed; the code rlca_safety_reduce runs). */
int rlca_safety_reduce_host(const rlca_env_config *cfg, const float *safety_records_host,
                            const float *eval_records_host, const int32_t *count_host, const uint8_t *role_mask_host,
                            int32_t episodes, int32_t world_begin, int32_t world_count, double *partials_host);

/* =====================================================================================
 * Progress metrics (csrc/rlca_progress.cu, DESIGN.md §9o): why robots time out or never finish, per episode of the
 * evaluation tracker above.
 *
 * A tick of a tracked episode (closed != meta_in.y) is folded unless it re-spawned the robot (flags.w).  A folded tick
 * takes d = pose_out.w (the distance to the goal the tick computed), the centre displacement
 * s = |(x, y)_out - (x, y)_in| and the heading change |wrap(theta_out - theta_in)|, and keeps per running episode:
 *   closest     the least d
 *   reference   the first folded tick sets ref = d and since = 0; a later one with d <= ref - progress_dist sets
 *               ref = d and since = 0, any other adds 1 to since (ticks since progress)
 *   still       a tick with s < still_dist is still; run counts consecutive still ticks (0 after a moving tick),
 *               still all still ticks of the episode
 *   rotation    the sum of the heading changes, radians
 *   near        another robot of the world, any, finished or parked included, had its centre strictly within
 *               block_dist of this robot's at the poses the tick ended at, on the last folded tick
 * Cause of an episode that ends with result 3 (time-out), and of an unfinished episode at the reduction:
 * 1 frozen (run >= window), else 2 stalled (since >= window), else 3 slow; + 4 when near is set.
 * ===================================================================================== */
typedef struct rlca_progress_params {
    int32_t window;              /* ticks; >= 1 */
    float progress_dist;         /* metres; finite, >= 0 */
    float still_dist;            /* metres per tick; finite, >= 0 */
    float block_dist;            /* metres; finite, >= 0 */
} rlca_progress_params;

/* Per-agent state, N rows; the caller zeroes running and counters before the first tick it tracks (all zero = no
 * folded tick yet: the next folded tick starts the episode's state).
 *   running    (N, 4) float  closest, progress reference, rotation, near (0 or 1) of the running episode
 *   counters   (N, 4) int32  ticks since progress, still run, still ticks, folded ticks of the running episode
 *   records    (N, episodes, 4) float, slot for slot the tracker's records: closest, rotation, still ticks, folded
 *              ticks (the counts held exactly below 2^24 ticks)
 *   causes     (N, episodes) uint8: the cause of a record whose episode timed out, 0 for every other record */
typedef struct rlca_progress_state {
    float *running_dev;
    int32_t *counters_dev;
    float *records_dev;
    uint8_t *causes_dev;
    int32_t episodes;
} rlca_progress_state;

/* One launch after each rlca_env_step and BEFORE that tick's rlca_eval_track, with the same cfg, state buffers and
 * io: reads the poses of state_in / state_out, the episode indices of state_in, io->flags_dev and the tracker's
 * closed / count (never written), so a tick belongs to the episode the tracker assigns it to and a record goes into
 * the slot the tracker fills next.  A tick that ends an episode writes the record (on a re-spawn tick from the state
 * the previous tick left) and zeroes the running state, as does any re-spawn.  It reads and writes nothing
 * rlca_safety_track does, so the two may run in either order.  RLCA_ERR_INVALID for a NULL pointer, robots_per_world
 * outside 1..64, episodes < 1 or different from the tracker's, a distance not finite or < 0, window < 1. */
int rlca_progress_track(const rlca_env_config *cfg, const rlca_progress_params *params,
                        const rlca_env_state *state_in, const rlca_env_state *state_out, const rlca_step_io *io,
                        const rlca_eval_state *ev, const rlca_progress_state *ps, void *stream);
/* The same from HOST buffers (pose (N,4) float; meta (N,4) int32; flags (N,4) uint8; the rest as the device state) by
 * serial loops over the same code; the outputs equal rlca_progress_track's bit for bit. */
int rlca_progress_track_host(const rlca_env_config *cfg, const rlca_progress_params *params,
                             const float *pose_in_host, const int32_t *meta_in_host, const float *pose_out_host,
                             const uint8_t *flags_host, const int32_t *closed_host, const int32_t *count_host,
                             int32_t episodes, float *running_host, int32_t *counters_host, float *records_host,
                             uint8_t *causes_host);

/* Per-world float64 partials of worlds [world_begin, world_begin + world_count), one thread per world in
 * agent-then-record order, no atomics: partials_dev (world_count, RLCA_PROGRESS_NPARTIALS).  The tracker's state gives
 * the number of records per agent, each record's result code and which agents are unfinished (fewer than `episodes`
 * records and open); an unfinished episode is classified from the running state with params->window.  With
 * role_mask_dev (N uint8) the partials are split as rlca_eval_reduce_split splits its own, partials_dev (world_count,
 * 2, RLCA_PROGRESS_NPARTIALS): row 0 over the agents with mask 0, row 1 over the others.  Every column is a sum;
 * totals add them in global world order. */
#define RLCA_PROGRESS_TIMEOUT_FROZEN 0          /* time-outs with cause frozen */
#define RLCA_PROGRESS_TIMEOUT_STALLED 1         /* ... stalled */
#define RLCA_PROGRESS_TIMEOUT_SLOW 2            /* ... slow */
#define RLCA_PROGRESS_TIMEOUT_ROBOT_NEAR 3      /* time-outs with robot near (+4) */
#define RLCA_PROGRESS_TIMEOUT_FOLDED 4          /* time-outs with at least one folded tick: the next two are over these */
#define RLCA_PROGRESS_TIMEOUT_SUM_CLOSEST 5     /* sum of closest */
#define RLCA_PROGRESS_TIMEOUT_SUM_CLOSEST_SQ 6  /* sum of closest squared */
#define RLCA_PROGRESS_UNFINISHED_FROZEN 7       /* the same seven over unfinished episodes */
#define RLCA_PROGRESS_UNFINISHED_STALLED 8
#define RLCA_PROGRESS_UNFINISHED_SLOW 9
#define RLCA_PROGRESS_UNFINISHED_ROBOT_NEAR 10
#define RLCA_PROGRESS_UNFINISHED_FOLDED 11
#define RLCA_PROGRESS_UNFINISHED_SUM_CLOSEST 12
#define RLCA_PROGRESS_UNFINISHED_SUM_CLOSEST_SQ 13
#define RLCA_PROGRESS_SUM_STILL_TICKS 14        /* over every recorded episode: still ticks */
#define RLCA_PROGRESS_SUM_TICKS 15              /* ... folded ticks */
#define RLCA_PROGRESS_REACHED 16                /* recorded episodes that reached the goal */
#define RLCA_PROGRESS_SUM_ROTATION 17           /* their rotation, radians */
#define RLCA_PROGRESS_SUM_ROTATION_SQ 18        /* ... squared */
#define RLCA_PROGRESS_NPARTIALS 19
int rlca_progress_reduce(const rlca_env_config *cfg, const rlca_progress_params *params,
                         const rlca_progress_state *ps, const rlca_eval_state *ev, const uint8_t *role_mask_dev,
                         int32_t world_begin, int32_t world_count, double *partials_dev, void *stream);
/* The same reduction from HOST buffers (no device needed; the code rlca_progress_reduce runs). */
int rlca_progress_reduce_host(const rlca_env_config *cfg, const rlca_progress_params *params,
                              const float *progress_records_host, const uint8_t *causes_host,
                              const float *running_host, const int32_t *counters_host,
                              const float *eval_records_host, const int32_t *count_host, const int32_t *open_host,
                              const uint8_t *role_mask_host, int32_t episodes, int32_t world_begin,
                              int32_t world_count, double *partials_host);

/* =====================================================================================
 * Sensor and actuation noise (csrc/rlca_noise.cu, DESIGN.md §9p): separate launches around the tick, issued only when
 * a run asks for noise; the tick itself and its outputs are untouched.
 *
 * Draws: Philox-4x32-10 under the key (seed lo, seed hi) of the counter
 *   (global agent = (world_offset + w) R + r, draw, element group, purpose | stream_id << 8)
 * with purposes 0xE1 range noise, 0xE2 dropout, 0xE3 action noise (one byte, so that no stream id shifted by 8 can
 * overlap them; the environment uses 1-5, the sampler 0x5A17).  `draw` is the caller's tick counter; `stream_id` tells
 * apart several env handles of one run (a mix component's index).  A uniform is the top 24 bits of a word times
 * 2^-24; a normal pair is Box-Muller on the words (w0, w1) or (w2, w3): u1 = ((w >> 8) + 1) 2^-24 in (0, 1],
 * u2 = (w >> 8) 2^-24, z = sqrt(-2 ln u1) (cos, sin)(2 pi u2), with the contract ln / sin / cos of rlca_common.cuh.
 * No draw depends on num_worlds, the launch shape or anything but the key and the counter.
 *
 * Scan (the newest frame of an (N, 3, beams) observation stack, normalised o = r / 6 - 0.5): element group g holds
 * beams 4g .. 4g + 3, one Philox call per group and purpose.  Per beam, r = (o + 0.5) range_max:
 *   dropout     u < dropout (float32 compare): the beam reads range_max (no return)
 *   range noise otherwise, a beam with a return (r < range_max) and range_sigma > 0 gets
 *               r' = clamp(fma(range_sigma, z, r), 0, range_max), written back as fma(r', 1/6, -0.5); a beam without a
 *               return stays as it is, so noise never makes a return
 * Action (N, 2): clip (v, w) to [v_min, v_max] x [w_min, w_max], multiply by max(fma(sigma, z, 1), 0) (z from group 0,
 * purpose 0xE3: z1 for v, z2 for w), clip again.  A gain never reverses a command, and a zero command stays zero.
 * ===================================================================================== */
typedef struct rlca_noise_params {
    float range_sigma;           /* metres; finite, >= 0 */
    float dropout;               /* probability a beam reads no return; in [0, 1] */
    float v_gain_sigma;          /* relative; finite, >= 0 */
    float w_gain_sigma;          /* relative; finite, >= 0 */
    uint64_t seed;
    uint32_t stream_id;          /* < 2^24 */
} rlca_noise_params;

/* In place on stack_dev (N, 3, beams) float, after a tick: perturbs the newest frame (slot 2) of every row, the two
 * older frames having been perturbed when they were newest.  A row whose flags_dev[4 a + 3] (was_reset) is set gets the
 * perturbed frame in all three slots, as the tick gives a re-spawned row three copies of its scan; flags_dev NULL means
 * every row is fresh (the first stack after a reset).  RLCA_ERR_INVALID for a NULL cfg, params or stack,
 * robots_per_world outside 1..64, num_worlds or beams < 1, world_offset < 0, a sigma negative or not finite, dropout
 * outside [0, 1] or stream_id >= 2^24. */
int rlca_noise_scan(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                    const unsigned char *flags_dev, float *stack_dev, void *stream);
/* Before a tick: the command the robots execute, action_out_dev (N, 2), from the command action_in_dev (N, 2), which is
 * never written.  The same argument checks, and action_in_dev / action_out_dev not NULL. */
int rlca_noise_action(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                      const float *action_in_dev, float *action_out_dev, void *stream);
/* The same from HOST buffers by serial loops over the same code; the outputs equal the kernels' bit for bit. */
int rlca_noise_scan_host(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                         const unsigned char *flags_host, float *stack_host);
int rlca_noise_action_host(const rlca_env_config *cfg, const rlca_noise_params *p, uint32_t draw,
                           const float *action_in_host, float *action_out_host);

/* =====================================================================================
 * Sensing and command latency (csrc/rlca_latency.cu, DESIGN.md §9q): separate launches around the tick, issued only
 * when a run asks for latency; the tick itself and its outputs are untouched.  One tick is dt = 0.1 s and every delay
 * is a whole number of ticks in 0 .. RLCA_LATENCY_MAX_DELAY.
 *
 * Delays: an agent draws its scan delay d in [scan_lo, scan_hi] and its command delay l in [cmd_lo, cmd_hi] when it
 * starts an episode (a row whose flags[4 a + 3], was_reset, is set, or every row when flags is NULL), and holds them
 * until its next one.  The draw is lo + (((hi - lo + 1) * (uint64)w0) >> 32), w0 the first word of Philox-4x32-10
 * under the key (seed lo, seed hi) of the counter
 *   (global agent = (world_offset + w) R + r, draw, 0, purpose | stream_id << 8)
 * with purposes 0xE4 scan, 0xE5 command (one byte; the environment uses 1-5, the sampler 0x5A17, noise 0xE1-0xE3).
 * `draw` is the caller's own counter of calls of that kind, 0, 1, 2, ...; it also picks the ring slot, draw mod
 * (hi + 1), so it must advance by one per call.  Everything is integer arithmetic and copies: the host twins equal the
 * kernels bit for bit, and no delay depends on num_worlds, the launch shape or anything but the key and the counter.
 *
 * Scan (after a tick and any re-layout, before scan noise): a ring of D = scan_hi + 1 frames per agent.  A fresh row
 * puts its newest frame in all D slots and redraws d; its stack, three copies of that frame, is left as it is.  Any
 * other row stores its newest frame in slot draw mod D and then reads slot (draw - d) mod D into the newest frame.  The
 * robot therefore reads the true frame of d calls earlier, or its episode's first frame while fewer than d calls have
 * passed; the stack's two older frames are what the tick shifted in, the frames delivered on the calls before.
 * Command (before noise and the tick, with the flags of the PREVIOUS tick, NULL on a run's first tick): a ring of
 * C = cmd_hi + 1 (v, w) pairs per agent.  A fresh row puts the issued command in all C slots and redraws l; then every
 * row stores the issued command (bit for bit, unclipped) in slot draw mod C and executes slot (draw - l) mod C: the
 * robot executes the command issued l calls earlier, or its episode's first command while fewer than l calls have
 * passed.  (Not a zero command: the tick's collision latch is cleared only by a move, so a re-spawned robot held still
 * would crash again on every tick.)
 * A kind whose hi is 0 is the identity: no launch, its ring and delay pointers may be NULL, and the action entry copies
 * the command to action_out (nothing when the two are the same buffer).
 * ===================================================================================== */
#define RLCA_LATENCY_MAX_DELAY 8
typedef struct rlca_latency_params {
    int32_t scan_lo, scan_hi;    /* ticks; 0 <= lo <= hi <= RLCA_LATENCY_MAX_DELAY */
    int32_t cmd_lo, cmd_hi;      /* ticks; the same */
    uint64_t seed;
    uint32_t stream_id;          /* < 2^24 */
} rlca_latency_params;

/* The state of one env handle's latency, in device memory for the device entries and host memory for the host twins;
 * N = num_worlds R rows of this config.  The caller allocates it and keeps it from call to call. */
typedef struct rlca_latency_state {
    float *scan_ring;            /* (N, scan_hi + 1, beams) float: the last scan_hi + 1 true frames per agent */
    float *cmd_ring;             /* (N, cmd_hi + 1, 2) float: the last cmd_hi + 1 issued commands per agent */
    uint8_t *scan_delay;         /* (N,) the scan delay of each agent's episode, ticks */
    uint8_t *cmd_delay;          /* (N,) the command delay of each agent's episode, ticks */
} rlca_latency_state;

/* In place on stack_dev (N, 3, beams) float, after a tick: the newest frame (slot 2) becomes the delayed frame.
 * RLCA_ERR_INVALID for a NULL cfg, params, state or stack, robots_per_world outside 1..64, num_worlds or beams < 1,
 * world_offset < 0, a delay range with lo < 0, lo > hi or hi > RLCA_LATENCY_MAX_DELAY, stream_id >= 2^24, or, with
 * scan_hi > 0, a NULL scan_ring or scan_delay. */
int rlca_latency_scan(const rlca_env_config *cfg, const rlca_latency_params *p, const rlca_latency_state *state,
                      uint32_t draw, const unsigned char *flags_dev, float *stack_dev, void *stream);
/* Before a tick: the command the robots execute, action_out_dev (N, 2), from the issued command action_in_dev (N, 2),
 * which is never written.  The same argument checks, with cmd_ring / cmd_delay for the command, and action_in_dev /
 * action_out_dev not NULL. */
int rlca_latency_action(const rlca_env_config *cfg, const rlca_latency_params *p, const rlca_latency_state *state,
                        uint32_t draw, const unsigned char *flags_dev, const float *action_in_dev,
                        float *action_out_dev, void *stream);
/* The same on HOST buffers (state included) by serial loops over the same code; the outputs equal the kernels'. */
int rlca_latency_scan_host(const rlca_env_config *cfg, const rlca_latency_params *p, const rlca_latency_state *state,
                           uint32_t draw, const unsigned char *flags_host, float *stack_host);
int rlca_latency_action_host(const rlca_env_config *cfg, const rlca_latency_params *p, const rlca_latency_state *state,
                             uint32_t draw, const unsigned char *flags_host, const float *action_in_host,
                             float *action_out_host);

/* =====================================================================================
 * Acceleration limits (csrc/rlca_dynamics.cu, DESIGN.md §9r): a separate launch just before the tick, issued only when
 * a run asks for limits; the tick itself and its outputs are untouched.
 *
 * Limits: an agent draws its linear limit a in [lin_lo, lin_hi] m/s^2 and its angular limit b in [ang_lo, ang_hi]
 * rad/s^2 when it starts an episode (a row whose flags[4 a + 3], was_reset, is set, or every row when flags is NULL),
 * and holds them until its next one.  With w0, w1 the first two words of Philox-4x32-10 under the key (seed lo, seed
 * hi) of the counter
 *   (global agent = (world_offset + w) R + r, draw, 0, 0xE6 | stream_id << 8)
 * (one-byte purpose; the environment uses 1-5, the sampler 0x5A17, noise 0xE1-0xE3, latency 0xE4-0xE5),
 * a = lin_lo + (lin_hi - lin_lo) u0 and b = ang_lo + (ang_hi - ang_lo) u1 with u = (w >> 8) 2^-24, in float32.
 * `draw` is the caller's own counter of calls, 0, 1, 2, ...
 *
 * Rule, per component, before the tick with the flags of the PREVIOUS tick (NULL on a run's first tick): the target is
 * what the tick would execute (a value with |x| > 3e38 or NaN becomes 0, then the clip to [v_min, v_max] / [w_min,
 * w_max]); prev is the agent's executed velocity of the last call, or (0, 0) for a fresh row and for a row whose
 * flags[4 a + 1] (crashed) is set; d = target - prev, s = limit * cfg->dt; the executed value is prev + s if d > s,
 * prev - s if d < -s, and the target itself otherwise.  It is written to action_out and stored in vel.  A kind whose
 * range is (0, 0) is off: its component is the target.  Limits that never bind therefore give the command the tick
 * would execute anyway, bit for bit.  Every function is shared by the kernel and the host twin, built without
 * contraction, so the two are equal bit for bit, and no limit depends on num_worlds, the launch shape or anything but
 * the key and the counter.
 * ===================================================================================== */
#define RLCA_DYNAMICS_MAX_ACCEL 100
typedef struct rlca_dynamics_params {
    float lin_lo, lin_hi;        /* m/s^2; (0, 0) off, else finite with 0 < lo <= hi <= RLCA_DYNAMICS_MAX_ACCEL */
    float ang_lo, ang_hi;        /* rad/s^2; the same */
    uint64_t seed;
    uint32_t stream_id;          /* < 2^24 */
} rlca_dynamics_params;

/* The state of one env handle's limits, in device memory for the device entry and host memory for the host twin;
 * N = num_worlds R rows of this config.  The caller allocates it and keeps it from call to call. */
typedef struct rlca_dynamics_state {
    float *vel;                  /* (N, 2) float: the (v, w) each agent executed on the last call */
    float *lin_limit;            /* (N,) float: the linear limit of each agent's episode, m/s^2 (0 when off) */
    float *ang_limit;            /* (N,) float: the angular limit, rad/s^2 (0 when off) */
} rlca_dynamics_state;

/* Before a tick: the command the robots execute, action_out_dev (N, 2), from the command action_in_dev (N, 2), which is
 * never written.  RLCA_ERR_INVALID for a NULL cfg, params, state, state buffer, action_in_dev or action_out_dev,
 * robots_per_world outside 1..64, num_worlds < 1, world_offset < 0, a range that is not (0, 0) and not finite with
 * 0 < lo <= hi <= RLCA_DYNAMICS_MAX_ACCEL, or stream_id >= 2^24. */
int rlca_dynamics_action(const rlca_env_config *cfg, const rlca_dynamics_params *p, const rlca_dynamics_state *state,
                         uint32_t draw, const unsigned char *flags_dev, const float *action_in_dev,
                         float *action_out_dev, void *stream);
/* The same on HOST buffers (state included) by a serial loop over the same code; the outputs equal the kernel's. */
int rlca_dynamics_action_host(const rlca_env_config *cfg, const rlca_dynamics_params *p,
                              const rlca_dynamics_state *state, uint32_t draw, const unsigned char *flags_host,
                              const float *action_in_host, float *action_out_host);

/* =====================================================================================
 * Localization error (csrc/rlca_localization.cu, DESIGN.md §9s): a separate launch after the tick, issued only when a
 * run asks for it; the tick itself, its state and its outputs are untouched, so success, crashes, rewards and every
 * tracker stay on the true state.  It changes only what the policy reads as gs: the local goal and the speed.
 *
 * Error process: each agent holds a pose-estimate error e = (ex, ey, etheta) in the world frame.  Each call, per
 * component, e <- rho e + kappa sigma xi with xi ~ N(0, 1), rho = exp(-dt / tau) and kappa = sqrt(1 - rho^2), both
 * computed once per call on the host in double and rounded to float (tau = 0: rho = 0, kappa = 1, white jitter;
 * tau = +inf: rho = 1, kappa = 0, and e is held as it is, a constant offset for the episode).  sigma is sigma_xy for
 * ex and ey and sigma_theta for etheta.  A row starts an episode (every row when flags is NULL, else a row whose
 * flags[4 a + 3], was_reset, of the tick just run is set): it draws sigma_xy in [xy_lo, xy_hi] and sigma_theta in
 * [theta_lo, theta_hi] and starts from the stationary distribution, e = sigma xi.
 *
 * What the policy reads, gs_out[a]: the local goal of goal_speed (the tick's own rule) at the believed pose
 * (x + ex, y + ey, theta + etheta) with dev_sincosf(theta + etheta), where a component whose error is exactly 0 keeps
 * the true value as it is (so zero error gives the tick's gs bit for bit, -0 included); and the speed gs_in[a].zw plus
 * N(0, v_sigma^2) and N(0, w_sigma^2) noise, fresh every call (a sigma of 0 keeps the value as it is).  The goal comes
 * from the env state's goal, the pose from its pose; gs_in is read for the speed only.
 *
 * Draws: with c = Philox-4x32-10 under the key (seed lo, seed hi) of the counter
 *   (global agent = (world_offset + w) R + r, draw, group, 0xE7 | stream_id << 8)
 * (one-byte purpose; the environment uses 1-5, the sampler 0x5A17, noise 0xE1-0xE3, latency 0xE4-0xE5, dynamics 0xE6),
 * group 0 gives the normals of ex, ey (Box-Muller of words 0, 1) and etheta, v (words 2, 3), and group 1 the normal of
 * w (words 0, 1) and the uniforms u = (w >> 8) 2^-24 of sigma_xy = xy_lo + (xy_hi - xy_lo) u2 and sigma_theta =
 * theta_lo + (theta_hi - theta_lo) u3.  Box-Muller is noise's (§9p).  `draw` is the caller's own counter of calls,
 * 0, 1, 2, ...  Every function is shared by the kernel and the host twin, built without contraction, so the two are
 * equal bit for bit, and no value depends on num_worlds, the launch shape or anything but the key and the counter.
 * ===================================================================================== */
typedef struct rlca_localization_params {
    float xy_lo, xy_hi;          /* m; finite, 0 <= lo <= hi */
    float theta_lo, theta_hi;    /* rad; the same */
    float tau;                   /* s; >= 0 or +inf */
    float v_sigma, w_sigma;      /* m/s, rad/s; finite, >= 0 */
    uint64_t seed;
    uint32_t stream_id;          /* < 2^24 */
} rlca_localization_params;

/* The state of one env handle's localization error, in device memory for the device entry and host memory for the
 * host twin; N = num_worlds R rows of this config.  The caller allocates it and keeps it from call to call. */
typedef struct rlca_localization_state {
    float *err;                  /* (N, 4) float: ex, ey, etheta of each agent, and a pad */
    float *sigma;                /* (N, 2) float: sigma_xy and sigma_theta of each agent's episode */
} rlca_localization_state;

/* After a tick (and any re-layout, latency and noise): the believed gs, gs_out_dev (N, 4), from the env state the tick
 * just wrote (state_env: pose_dev and goal_dev are read, nothing is written) and the true gs_in_dev (N, 4).  gs_in_dev
 * may equal gs_out_dev (in place).  RLCA_ERR_INVALID for a NULL cfg, params, state, state buffer, state_env, pose or
 * goal buffer, gs_in_dev or gs_out_dev, robots_per_world outside 1..64, num_worlds < 1, world_offset < 0, a sigma
 * range that is not finite with 0 <= lo <= hi, a speed sigma that is not finite and >= 0, tau that is not >= 0 or +inf,
 * or stream_id >= 2^24. */
int rlca_localization_observe(const rlca_env_config *cfg, const rlca_localization_params *p,
                              const rlca_localization_state *state, uint32_t draw, const unsigned char *flags_dev,
                              const rlca_env_state *state_env, const float *gs_in_dev, float *gs_out_dev,
                              void *stream);
/* The same on HOST buffers (state and env state included) by a serial loop over the same code; the outputs equal the
 * kernel's. */
int rlca_localization_observe_host(const rlca_env_config *cfg, const rlca_localization_params *p,
                                   const rlca_localization_state *state, uint32_t draw,
                                   const unsigned char *flags_host, const rlca_env_state *state_host,
                                   const float *gs_in_host, float *gs_out_host);

/* =====================================================================================
 * Dynamic-window baseline (DESIGN.md §9u), csrc/rlca_dwa.cu: a sensor-level classical controller that reads exactly
 * what the policy reads, so it can stand in the policy's slot of an evaluation (Fox, Burgard, Thrun 1997).
 *
 * Inputs, N = num_worlds R rows: stack (N, 3, beams), the policy's scan FIFO, of which only frame 2 (the newest) is
 * read, a beam's range being (s + 0.5) range_max and a beam at range_max having no return; gs (N, 4), the local goal
 * x, y in the robot frame and the speed v, w the policy reads; beam_cos_sin (beams, 2), each beam's unit vector in the
 * robot frame (the env's own beam angles).  Per robot, with the disc of radius rho = radius and constant-(v, w) arcs:
 *   window     v_samples x w_samples candidates over [v0 - accel dt, v0 + accel dt] n [v_min, v_max] and the same for
 *              w with angular_accel, (v0, w0) = the gs speed clamped into the action box; a limit of 0 takes the
 *              whole box.  Sample i of n is lo + (hi - lo) (i / (n - 1)), hi exactly at i = n - 1, the midpoint at
 *              n = 1; candidate c = iv w_samples + iw.
 *   clearance  the arc length the disc drives before it first touches a return within reach (v_hi horizon + rho), in
 *              closed form (straight below |w| = 1e-6 rad/s), capped at v horizon; clearance_cap when v = 0; and 0 for
 *              every candidate when any return lies within rho.
 *   admissible clearance > 0 and clearance >= v dt + v^2 / (2 brake).
 *   score      heading_weight (1 - |bearing of the goal from the pose after heading_time| / pi)
 *              + clearance_weight min(clearance, cap) / cap + speed_weight v / v_max.
 * The action is the admissible candidate of highest score, the lowest index among equals, with status 0; with none,
 * (0, 0) and status 1.  One warp per robot; every function is shared with the host entry and the file is built
 * without contraction, so the two are equal bit for bit.
 * ===================================================================================== */
#define RLCA_DWA_MAX_CANDIDATES 1024
#define RLCA_DWA_MAX_BEAMS 512
typedef struct rlca_dwa_params {
    int32_t v_samples, w_samples;    /* candidate grid over the window, both >= 1, product <= RLCA_DWA_MAX_CANDIDATES */
    float radius;                    /* disc radius of the robot, m */
    float horizon;                   /* arc simulated per candidate, s */
    float heading_time;              /* the goal bearing is scored from the pose predicted after this, s */
    float accel, angular_accel;      /* window half-widths are accel*dt, angular_accel*dt; 0 = the whole action box */
    float brake;                     /* admissible iff clearance >= v*dt + v^2 / (2 brake), m/s^2 */
    float heading_weight, clearance_weight, speed_weight;
    float clearance_cap;             /* clearance is scored as min(clearance, cap) / cap, m */
} rlca_dwa_params;

/* The action (N, 2) and status (N) of every robot, on `stream`.  RLCA_ERR_INVALID for a NULL pointer, robots_per_world
 * or num_worlds < 1, beams outside 2..RLCA_DWA_MAX_BEAMS, a config without finite range_max, dt, v_max > 0 and
 * v_min <= v_max, w_min <= w_max, a sample count < 1 or a grid above RLCA_DWA_MAX_CANDIDATES, a radius, horizon, brake
 * or cap that is not finite and > 0, or a heading_time, limit or weight that is not finite and >= 0. */
int rlca_dwa_action(const rlca_env_config *cfg, const rlca_dwa_params *p, const float *beam_cos_sin_dev,
                    const float *stack_dev, const float *gs_dev, float *action_dev, int32_t *status_dev, void *stream);
/* The same on HOST buffers by a serial loop over the same code; equal to rlca_dwa_action bit for bit.  clearance_host
 * and score_host, each (N, v_samples w_samples) or NULL, receive every candidate's clearance and score (the score of
 * inadmissible candidates included). */
int rlca_dwa_action_host(const rlca_env_config *cfg, const rlca_dwa_params *p, const float *beam_cos_sin_host,
                         const float *stack_host, const float *gs_host, float *action_host, int32_t *status_host,
                         float *clearance_host, float *score_host);

/* =====================================================================================
 * Global planner (DESIGN.md §9w), csrc/rlca_plan.cu: geodesic fields to each robot's goal, line-of-sight waypoints as
 * the policy's local goal, and the geodesic length of every episode.
 *
 * Graph: the traversable cells (rl_collision_avoidance_b200/planner.py: no non-free cell within r_c + res sqrt(2) / 2
 * of the cell's centre, cells outside the grid non-free), 8-neighbour moves of cost 70 (orthogonal) and 99 (diagonal,
 * allowed only when both orthogonal neighbours are traversable).  D(c) is the least path cost from cell c to a row's
 * goal entry cell; 0xFFFFFFFF where there is no path.  Cells are the tick's: cx = floor(x ppm) + origin_cx, the same
 * for y; an index is cy grid_w + cx.
 *   goal entry   the goal's cell if traversable, else the traversable cell of its 5 x 5 neighbourhood whose centre is
 *                nearest the goal point (float32, cell units), ties in row-major order; none = no plan
 *   robot entry  the robot's cell if it lies in the goal entry's component, else the cell of least D in its 5 x 5
 *                neighbourhood, ties in row-major order; none = no plan
 *   visible      every cell the closed segment from the robot's centre to a target point meets is traversable, but
 *                for cells within chessboard distance 1 of either end point's cell (a float32 supercover walk, column
 *                by column in cell units)
 * ===================================================================================== */
/* shared memory of one CTA on sm_90a (227 KB) at 4 bytes per cell: the largest component rectangle a field may span */
#define RLCA_PLAN_MAX_CELLS 58112

/* The planning graph of a map: label (grid_h, grid_w) int32, the component of each traversable cell and -1 elsewhere;
 * rects (num_components, 4) int32, each component's bounding rectangle cx0, cy0, cx1, cy1 (inclusive); max_area the
 * largest rectangle's cell count.  Device pointers for the device entries, host pointers for the host twins. */
typedef struct rlca_plan_tables {
    int32_t num_components;
    int32_t max_area;            /* 1..RLCA_PLAN_MAX_CELLS */
    const int32_t *label;
    const int32_t *rects;
} rlca_plan_tables;

/* RLCA_OK when host tables hold what the device entries rely on: labels in -1..num_components - 1, every rectangle
 * non-empty, inside the grid and at most max_area cells, every labelled cell inside its component's rectangle,
 * max_area in 1..RLCA_PLAN_MAX_CELLS.  RLCA_ERR_INVALID otherwise.  Run it on the host copy before uploading. */
int rlca_plan_tables_check(const rlca_env_config *cfg, const rlca_plan_tables *tables_host);

/* The planner's per-row state, N = num_worlds R rows; device pointers for the device entries, host pointers for the
 * host twins.  The caller sets entry to -1 before the first rlca_plan_fields and zeroes status_count.
 *   entry         (N) int32 goal entry cell of the row's field, -1 = no plan
 *   rect          (N, 4) int32 the field's rectangle (its component's)
 *   field         (N, max_area) uint32 D over the rectangle, row-major, row width cx1 - cx0 + 1
 *   list          (N + 1) int32 the rows the last rlca_plan_fields re-planned: count, then the rows (device: in any
 *                 order; host: ascending)
 *   status        (N) uint8 of the last rlca_plan_waypoints: 0 goal visible, 1 waypoint, 2 no plan
 *   status_count  (N, 3) int32, incremented per row and status by every rlca_plan_waypoints
 *   length        (N) float geodesic length L = D(start entry) res / 70 of the running episode, -1 = no path
 *   records       (N, episodes) float L of the tracker's records, slot for slot
 * The tracker fields (length, records, episodes) are read by rlca_plan_track and rlca_plan_reduce only. */
typedef struct rlca_plan_state {
    int32_t *entry;
    int32_t *rect;
    uint32_t *field;
    int32_t *list;
    uint8_t *status;
    int32_t *status_count;
    float *length;
    float *records;
    int32_t episodes;
} rlca_plan_state;

/* Re-plan the rows whose goal entry (from state->goal_dev) differs from ps->entry: their field over the component's
 * rectangle and their entry and rect.  A goal with no entry sets entry -1.  RLCA_ERR_INVALID for a NULL pointer,
 * robots_per_world outside 1..64, num_worlds < 1, a config without a map, tables with no component or max_area outside
 * 1..RLCA_PLAN_MAX_CELLS. */
int rlca_plan_fields(const rlca_env_config *cfg, const rlca_plan_tables *tables, const rlca_plan_state *ps,
                     const rlca_env_state *state, void *stream);
/* The same on HOST buffers by a serial loop over the same code; equal to rlca_plan_fields bit for bit.  Also
 * RLCA_ERR_INVALID for what rlca_plan_tables_check rejects. */
int rlca_plan_fields_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                          const rlca_plan_state *ps_host, const rlca_env_state *state_host);

/* gs_out (N, 4) from the poses and goals of `state` (the state a tick just wrote), the fields and gs_in (N, 4), the gs
 * the tick wrote: status 0 (goal visible) and 2 (no plan) copy gs_in; status 1 writes goal_speed of the pose and the
 * centre of the farthest visible cell of a chain of up to 64 steepest-descent steps from the robot's entry cell (ties
 * E, N, W, S, NE, NW, SW, SE; the first chain cell when none is visible; the entry cell itself when it is the goal
 * entry), with gs_in's speed half.  RLCA_ERR_INVALID as rlca_plan_fields, and for gs_in equal to gs_out. */
int rlca_plan_waypoints(const rlca_env_config *cfg, const rlca_plan_tables *tables, const rlca_plan_state *ps,
                        const rlca_env_state *state, const float *gs_in_dev, float *gs_out_dev, void *stream);
int rlca_plan_waypoints_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                             const rlca_plan_state *ps_host, const rlca_env_state *state_host, const float *gs_in_host,
                             float *gs_out_host);

/* Training with the planner (DESIGN.md §9x): rlca_plan_waypoints' rows (gs_out, status, status_count, the same rule)
 * and, in the same launch, a geodesic progress reward.  Per row, from the state the tick (and any re-layout) left:
 *   psi = 0 for status 0 and 2; for status 1, with w the waypoint (the centre of chain cell c_w),
 *   psi = (sqrtf(fmaf(dx, dx, dy dy)) + D(c_w) res / 70) - pose.w     (dx, dy = w - pose, float32; D res / 70 as in
 *         the geodesic length), so that pose.w + psi is the distance to the waypoint plus its geodesic length
 * With flags (N, 4) of the tick (after rlca_layout_*respawn): flags.x == 0 (a non-terminal tick): reward += progress_gain
 * (psi_prev - psi) in place; flags.x != 0: the reward is left as it is, and where the tick wrote the row's eplog
 * (flags.z != 0) its return column eplog[8 a + 2] += progress_gain (psi_start - psi_prev) when eplog is not NULL.  Then
 * psi_prev = psi, and psi_start = psi where flags.w != 0.  flags NULL (a run's start; reward and eplog unused): psi_prev
 * = psi_start = psi for every row.  psi_prev and psi_start (N) float are the caller's, as are reward (N) and eplog
 * (N, 8).  gs_in may equal gs_out (in place).  RLCA_ERR_INVALID as rlca_plan_waypoints, for a NULL psi buffer, psi_prev
 * equal to psi_start, or flags without reward.  The host twin equals the kernel bit for bit. */
int rlca_plan_shape(const rlca_env_config *cfg, const rlca_plan_tables *tables, const rlca_plan_state *ps,
                    float *psi_prev_dev, float *psi_start_dev, const rlca_env_state *state, const uint8_t *flags_dev,
                    float *reward_dev, float *eplog_dev, const float *gs_in_dev, float *gs_out_dev, void *stream);
int rlca_plan_shape_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                         const rlca_plan_state *ps_host, float *psi_prev_host, float *psi_start_host,
                         const rlca_env_state *state_host, const uint8_t *flags_host, float *reward_host,
                         float *eplog_host, const float *gs_in_host, float *gs_out_host);

/* After rlca_plan_fields of a tick and BEFORE that tick's rlca_eval_track, with the tick's state_in, state_out and
 * flags: an episode the tracker tracks (closed != meta_in.y) that ends (flags.z != 0) writes its length into the record
 * slot the tracker fills next; then a re-spawn (flags.w) sets length from the init pose (state_out acc.zw) and the row's
 * current field.  flags NULL (a run's start, state_in unused): every row's length from its init pose.  RLCA_ERR_INVALID
 * as rlca_plan_fields, for episodes < 1 or different from the tracker's, or a NULL buffer. */
int rlca_plan_track(const rlca_env_config *cfg, const rlca_plan_tables *tables, const rlca_plan_state *ps,
                    const rlca_env_state *state_in, const rlca_env_state *state_out, const uint8_t *flags_dev,
                    const rlca_eval_state *ev, void *stream);
int rlca_plan_track_host(const rlca_env_config *cfg, const rlca_plan_tables *tables_host,
                         const rlca_plan_state *ps_host, const rlca_env_state *state_in_host,
                         const rlca_env_state *state_out_host, const uint8_t *flags_host, const int32_t *closed_host,
                         const int32_t *count_host, int32_t episodes);

/* Per-world float64 partials of worlds [world_begin, world_begin + world_count), one thread per world (and role) in
 * agent-then-record order, no atomics: partials_dev (world_count, RLCA_PLAN_NPARTIALS), or (world_count, 2, ...) split
 * by an agent mask as rlca_eval_reduce_split splits.  Over recorded episodes that reached the goal with a path, with
 * the straight-line metric's goal radius: extra = path - max(L - goal_radius, 0). */
#define RLCA_PLAN_REACHED 0          /* episodes with result 1 and a path */
#define RLCA_PLAN_SUM_LENGTH 1       /* sum of their L */
#define RLCA_PLAN_SUM_EXTRA 2        /* sum, sum of squares of their extra geodesic distance */
#define RLCA_PLAN_SUM_EXTRA_SQ 3
#define RLCA_PLAN_NO_PATH 4          /* recorded episodes, any result, whose start had no path to the goal */
#define RLCA_PLAN_NPARTIALS 5
int rlca_plan_reduce(const rlca_env_config *cfg, const rlca_plan_state *ps, const rlca_eval_state *ev,
                     int32_t world_begin, int32_t world_count, double *partials_dev, void *stream);
int rlca_plan_reduce_split(const rlca_env_config *cfg, const rlca_plan_state *ps, const rlca_eval_state *ev,
                           const uint8_t *mask_dev, int32_t world_begin, int32_t world_count, double *partials_dev,
                           void *stream);
/* The same from HOST buffers: geo_records (N, episodes), the tracker's records and count, mask NULL or (N). */
int rlca_plan_reduce_host(const rlca_env_config *cfg, const float *geo_records_host, const float *eval_records_host,
                          const int32_t *count_host, const uint8_t *mask_host, int32_t episodes, int32_t world_begin,
                          int32_t world_count, double *partials_host);

/* sizeof(rlca_env_config) as compiled, so bindings can verify their struct layout. */
int rlca_sizeof_env_config(void);

const char *rlca_last_error(void);
const char *rlca_version(void);

#ifdef __cplusplus
}
#endif
#endif /* RLCA_H */
