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
 * deterministic == 1 -> action = mean (generate_action_no_sampling, model/ppo.py:84-107);
 * deterministic == 2 -> action_dev is an INPUT and only its logprob is evaluated (evaluate_actions, model/net.py:72-80). */
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

/* sizeof(rlca_env_config) as compiled, so bindings can verify their struct layout. */
int rlca_sizeof_env_config(void);

const char *rlca_last_error(void);
const char *rlca_version(void);

#ifdef __cplusplus
}
#endif
#endif /* RLCA_H */
