/*
 * pulse_b200.h -- C ABI of the GPU-native PULSE hot path (libpulse_b200.so, H100 / sm_90a).
 *
 * Boundary rules (SURVEY.md section 8b):
 *   - plain C types only: device pointers, element strides, sizes, a cudaStream_t passed as void*;
 *   - every buffer is owned by the caller (torch tensors or Isaac Gym gymtorch views); nothing is
 *     allocated on the device inside the library;
 *   - no hidden synchronisation: kernels are enqueued on the caller's stream and the call returns;
 *   - every entry point returns 0 on success or a negative pulse_status; the message is available
 *     from pulse_last_error() (thread-local).  No exceptions cross the boundary;
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     PULSE_ERR_CUDA;
 *   - ONE device per process (the reference's model: one Isaac Gym sim per process, run_hydra.py:117-131): launch attributes,
 *     the SM count and the persistent-grid sizes are cached per process on first use, so a process must not drive two
 *     different devices through this library; calls are made from one host thread per process, on the caller's stream.
 *
 * Each entry point cites the reference interface (file:line under the PULSE tree) it replaces.
 */
#ifndef PULSE_B200_H_
#define PULSE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PULSE_ABI_VERSION 3

enum pulse_status {
  PULSE_OK = 0,
  PULSE_ERR_ARG = -1,    /* null pointer / bad size / bad stride / misaligned table */
  PULSE_ERR_CUDA = -2,   /* CUDA runtime error (launch, no device, ...) */
  PULSE_ERR_UNSUPPORTED = -3
};

#define PULSE_NUM_BODIES 24        /* SMPL humanoid rigid bodies (smpl_humanoid.xml)        */
#define PULSE_NUM_DOF 69           /* 23 joints x 3                                           */
#define PULSE_BODY_STATE_W 13      /* pos3 quat4(xyzw) linvel3 angvel3, humanoid.py:215-222  */
#define PULSE_SELF_OBS 358         /* humanoid.py:1675-1731                                   */
#define PULSE_TASK_OBS_V6 576      /* humanoid_im.py:1328-1378                                */
#define PULSE_IM_OBS (PULSE_SELF_OBS + PULSE_TASK_OBS_V6)
#define PULSE_AMP_OBS 196          /* humanoid_amp.py:924-969 with dof_subset                 */
#define PULSE_FRAME_REC 312        /* packed per-frame record: pos72 | rot96 | vel72 | angvel72 */
#define PULSE_AUX_REC 240          /* packed per-frame record: lrs96 | dvs69 | aa72 | pad3    */

int pulse_abi_version(void);
const char* pulse_last_error(void);
/* Number of kernels this library has launched in the calling process (bench.py "gpu_launches"). */
int64_t pulse_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * MotionLib tables.  Replaces the device-resident buffers MotionLibBase.load_motions builds
 * (phc/utils/motion_lib_base.py:287-316) with two packed per-frame records so that one query
 * gathers one contiguous 1248-byte row per frame instead of rows of six separate tables.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pulse_motionlib pulse_motionlib_t;

typedef struct {
  /* reference tables, device pointers, contiguous fp32 / int64 (motion_lib_base.py:297-315) */
  const float* gts;   /* [F,24,3] */
  const float* grs;   /* [F,24,4] */
  const float* lrs;   /* [F,24,4] */
  const float* gvs;   /* [F,24,3] */
  const float* gavs;  /* [F,24,3] */
  const float* dvs;   /* [F,23,3] */
  const float* motion_aa; /* [F,72] (may be NULL -> zeros) */
  const float* lengths;         /* [M] _motion_lengths */
  const float* dt;              /* [M] _motion_dt */
  const int64_t* num_frames;    /* [M] _motion_num_frames */
  const int64_t* length_starts; /* [M] length_starts */
  int64_t total_frames;         /* F */
  int64_t num_motions;          /* M */
  /* caller-allocated packed outputs, 16-byte aligned, filled by pulse_motionlib_create */
  float* frame_rec;   /* [F, PULSE_FRAME_REC] */
  float* aux_rec;     /* [F, PULSE_AUX_REC]   */
} pulse_motionlib_desc_t;

/* Packs the tables (one kernel on `stream`) and returns a host-side handle that keeps the pointers.
 * The per-motion arrays and the packed records must outlive the handle. */
int pulse_motionlib_create(const pulse_motionlib_desc_t* desc, void* stream, pulse_motionlib_t** out);
int pulse_motionlib_destroy(pulse_motionlib_t* lib);

/* MotionLibBase.get_motion_state(motion_ids, motion_times, offset)  motion_lib_base.py:434-517
 * (+ _calc_frame_blend :546-556, _local_rotation_to_dof_smpl :561-564).  Any output may be NULL. */
typedef struct {
  const int64_t* motion_ids;   /* [n] */
  const float* motion_times;   /* [n] */
  const float* offset;         /* [n,3] or NULL */
  float* root_pos;      /* [n,3]   */
  float* root_rot;      /* [n,4]   */
  float* dof_pos;       /* [n,69]  */
  float* root_vel;      /* [n,3]   */
  float* root_ang_vel;  /* [n,3]   */
  float* dof_vel;       /* [n,69]  */
  float* motion_aa;     /* [n,72]  */
  float* rg_pos;        /* [n,24,3] */
  float* rb_rot;        /* [n,24,4] */
  float* body_vel;      /* [n,24,3] */
  float* body_ang_vel;  /* [n,24,3] */
  int64_t* frame_idx0;  /* [n] (diagnostic: _calc_frame_blend) */
  int64_t* frame_idx1;  /* [n] */
  float* blend;         /* [n] */
} pulse_motion_query_t;
int pulse_motion_state(const pulse_motionlib_t* lib, const pulse_motion_query_t* q, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused HumanoidIm post-physics step: reward(t) -> reset(t) -> observation(t+dt) in ONE kernel.
 * Replaces, for the default task configuration (obs_v 6, self_obs_v 1, full-body reward, 24 tracked
 * bodies, upright start, local_root_obs, root_height_obs):
 *   HumanoidIm._compute_reward        phc/env/tasks/humanoid_im.py:853-919  (compute_imitation_reward :1543-1574)
 *   HumanoidIm._compute_reset         humanoid_im.py:1119-1192              (compute_humanoid_im_reset :1600-1628)
 *   HumanoidIm._compute_observations  humanoid_im.py:677-706, _compute_task_obs :708-851
 *                                     (compute_imitation_observations_v6 :1328-1378)
 *   Humanoid._compute_humanoid_obs    phc/env/tasks/humanoid.py:1137-1213   (compute_humanoid_observations_smpl_max :1675-1731)
 *   and the two MotionLib queries behind _get_state_from_motionlib_cache (humanoid_im.py:950-964).
 * `progress_buf` is the value AFTER the reference's `progress_buf += 1` (humanoid.py:1317).
 * ---------------------------------------------------------------------------------------------- */
#define PULSE_STEP_REWARD 1u
#define PULSE_STEP_RESET 2u
#define PULSE_STEP_OBS 4u
#define PULSE_STEP_ALL 7u
#define PULSE_STEP_ADVANCE 8u   /* ABI 2: the kernel itself performs `progress_buf += 1` (humanoid.py:1317) through progress_rw before using it */

typedef struct {
  /* simulator state (Isaac Gym views, read-only) */
  const float* body_state;   /* rigid body state; env e, body j at body_state + e*body_env_stride + j*13 */
  int64_t body_env_stride;   /* floats between envs = bodies_per_env*13 (humanoid.py:215-222) */
  const float* dof_vel;      /* dof velocity; element k of env e at dof_vel + e*dof_env_stride + k*dof_elem_stride */
  int64_t dof_env_stride;    /* Isaac Gym dof-state view: dofs_per_env*2, elem stride 2 (humanoid.py:207-210) */
  int64_t dof_elem_stride;
  const float* dof_force;    /* [N,69] dof_force_tensor (humanoid.py:189-190); NULL disables the power term */
  int64_t dof_force_stride;
  /* optional env subset: warp i processes env env_ids[i] (reset path, humanoid_im.py:677-681); NULL = envs 0..n-1 */
  const int64_t* env_ids;
  /* task buffers (read-only) */
  const int64_t* progress_buf;      /* [N] */
  const int64_t* motion_ids;        /* [N] _sampled_motion_ids */
  const float* motion_start_times;  /* [N] */
  const float* motion_start_offset; /* [N] _motion_start_times_offset */
  const float* global_offset;       /* [N,3] */
  const int32_t* cycle_counter;     /* [N] or NULL */
  const int64_t* reset_buf_in;      /* unused by the reference's formula (kept for signature parity); may be NULL */
  const float* termination_distances; /* [24] _termination_distances (humanoid_im.py:1166-1186) */
  uint32_t reset_body_mask;         /* bit j set = body j in reset_bodies (env_im.yaml:38) */
  uint32_t flags;                   /* PULSE_STEP_* */
  float dt;                         /* control dt, fp32(2/60) */
  float k_pos, k_rot, k_vel, k_ang_vel, w_pos, w_rot, w_vel, w_ang_vel; /* reward_specs humanoid_im.py:55 */
  float power_coefficient;          /* humanoid_im.py:91; used when dof_force != NULL */
  int32_t cycle_motion;             /* 0: pass_time = t >= motion_len; 1: progress >= max_episode_length-1 */
  int64_t max_episode_length;
  int32_t enable_early_termination;
  int32_t use_mean_reset;           /* flags.im_eval && !strict_eval (humanoid_im.py:1606) */
  /* outputs (any may be NULL when its stage is disabled) */
  float* obs_buf;        /* [N, obs_stride], first 934 floats written */
  int64_t obs_stride;
  float* self_obs_buf;   /* [N,358] optional copy (humanoid_im.py:683) */
  float* rew_buf;        /* [N] */
  float* reward_raw;     /* [N, raw_stride]: pos, rot, vel, ang_vel (, power) */
  int64_t raw_stride;
  int64_t* reset_buf;    /* [N] */
  int64_t* terminate_buf;/* [N] */
  uint8_t* pass_time;    /* [N] optional: t >= motion_len mask (needed by the cycle_motion host path) */
  float* ref_body_pos;   /* [N,24,3] optional (humanoid_im.py:835-848) */
  float* ref_body_vel;   /* [N,24,3] optional */
  float* ref_body_rot;   /* [N,24,4] optional */
  float* ref_dof_pos;    /* [N,69]   optional (costs 2 extra 960-byte gathers per env) */
  /* ---- ABI 2 ---- */
  const int32_t* env_count;        /* optional DEVICE-side length of env_ids (the compacted list pulse_reset_ref_state writes): only the
                                      first min(num_envs, *env_count) entries are processed -- no host read of the count is ever needed */
  const int32_t* recovery_counter; /* [N] or NULL.  HumanoidImGetup._compute_reset (humanoid_im_getup.py:203-210): for envs with
                                      recovery_counter > 0 the reset / terminate outputs are forced to 0 and progress_buf is decremented
                                      (through progress_rw) BEFORE the observation time is formed */
  int64_t* progress_rw;            /* writable alias of progress_buf; required with recovery_counter */
  float* fdones_out;               /* [N] optional float copy of reset_buf (the experience buffer's `dones`, amp_agent.py:383) */
} pulse_im_step_args_t;
/* num_envs = number of envs processed (= len(env_ids) when env_ids is given). */
int pulse_im_step(const pulse_motionlib_t* lib, const pulse_im_step_args_t* args, int64_t num_envs, void* stream);

/* Tracked-body observation of the fused step (HumanoidImZ, env_pulse_im.yaml: trackBodies [Head, L_Hand, R_Hand], obs_v 6).
 * pulse_im_track_step is pulse_im_step (same arguments, flags, env list, side buffers, full-body reward and reset) whose observation
 * row is [358 self | task observation of the K tracked bodies], block-major as compute_imitation_observations_v6 / _v7
 * (humanoid_im.py:1328-1413) over the bodies in `_track_bodies_id` order:
 *   version 6: dp | rot6(dq) | dv | dw | R(p_ref - p_root) | rot6(q_ref)   358 + 24 K floats
 *   version 7: dp | dv | R(p_ref - p_root)                                  358 + 9 K floats
 * obs_stride must be at least that width; the row's columns beyond it are not written. */
typedef struct {
  int8_t rank[24];     /* rank[j]: position of body j in _track_bodies_id, -1 = untracked; the ranks are a permutation of 0..K-1 */
  int32_t num_track;   /* K in [1, 24] */
  int32_t version;     /* 6 or 7 */
} pulse_im_track_t;
int pulse_im_track_step(const pulse_motionlib_t* lib, const pulse_im_step_args_t* args, const pulse_im_track_t* track, int64_t num_envs,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * AMP observation + history shift.
 *   HumanoidAMP._update_hist_amp_obs      phc/env/tasks/humanoid_amp.py:622-630
 *   HumanoidAMP._compute_amp_observations humanoid_amp.py:632-667 (build_amp_observations_smpl :924-969,
 *                                         dof_to_obs_smpl humanoid.py:1436-1446), has_dof_subset = True.
 * amp_obs_buf is [N, num_steps, 196], index 0 = newest; in place: buf[:,1:] <- buf[:,:-1]; buf[:,0] <- new.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* body_state; int64_t body_env_stride;
  const float* dof_pos; const float* dof_vel; int64_t dof_env_stride; int64_t dof_elem_stride;
  float* amp_obs_buf;   /* [N, num_steps, 196] */
  int32_t num_steps;    /* numAMPObsSteps (env_im.yaml:31) */
  int32_t shift_history;/* 1: shift then write slot 0;  0: write slot 0 only */
} pulse_amp_obs_args_t;
int pulse_amp_obs(const pulse_amp_obs_args_t* args, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Rollout glue of AMPAgent.play_steps (phc/learning/amp_agent.py:341-439), written straight into the experience-buffer slices.
 *   pulse_policy_post   get_action_values' sampling (common_agent.py:262-288; ModelA2CContinuousLogStd [rl_games]): action = mu +
 *                       exp(logstd) * eps, neglogp, de-normalised value (running_mean_std.py:84-87), optional PD targets
 *                       (Humanoid._action_to_pd_targets, humanoid.py:1392-1394).  eps: injected, or Philox4x32-10(seed,
 *                       row, *rng_offset + rng_step) drawn in the kernel (a device-side offset keeps CUDA-graph replays fresh;
 *                       the index layout per row is listed with the other Philox planes below).  1 <= num_actions <= 256.
 *   pulse_value_post    next_values = unnormalise(critic(next obs)) * (1 - terminated)   (amp_agent.py:396-398)
 *   pulse_amp_obs_row   AMP observation row of this step = [current W | first (steps-1)*W floats of the previous row], written
 *                       into its experience slice (humanoid_amp.py:622-667 + amp_agent.py:385); W = amp_width (196 by default, 195
 *                       without the root height), the heading of remove_base_rot(q0) with remove_base_rot set
 *   pulse_bump_counter  *counter += by (one thread): advances the device-side RNG offset once per iteration
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* mu; int64_t ld_mu;            /* [rows, A] actor head output */
  const float* logstd;                       /* [A] */
  const float* eps; int64_t ld_eps;          /* [rows, A] injected standard-normal draws, or NULL -> Philox */
  uint64_t seed; const uint64_t* rng_offset; uint64_t rng_step;
  int32_t num_actions; int32_t reserved;
  float* actions; int64_t ld_actions;        /* out */
  float* neglogp; int64_t ld_neglogp;        /* out, element stride */
  float* mus_out; int64_t ld_mus;            /* optional copy of mu (NULL when the head GEMM already wrote the experience slice) */
  const float* value; int64_t ld_value;      /* [rows] normalised critic output (optional) */
  const double* value_mean; const double* value_var; float value_eps; int32_t reserved2;   /* RunningMeanStd of the value (NULL = identity) */
  float* values_out; int64_t ld_values;      /* optional */
  const float* pd_offset; const float* pd_scale; float* pd_targets; int64_t ld_pd;   /* optional */
} pulse_policy_post_args_t;
int pulse_policy_post(const pulse_policy_post_args_t* args, int64_t rows, void* stream);
int pulse_value_post(const float* value, int64_t ld_value, const double* mean, const double* var, float eps, const int64_t* terminate,
                     float* out, int64_t ld_out, int64_t rows, void* stream);
typedef struct {
  const float* body_state; int64_t body_env_stride;
  const float* dof_pos; const float* dof_vel; int64_t dof_env_stride; int64_t dof_elem_stride;
  const float* prev; int64_t ld_prev;        /* previous step's row of every env (floats between envs) */
  float* out; int64_t ld_out;                /* this step's row */
  int32_t num_steps; int32_t reserved;
  int32_t* fresh;                            /* [N] optional flags set by pulse_reset_ref_state; cleared here */
  const float* fresh_rows;                   /* [N, num_steps, amp_width] the back-filled rows of reset envs */
  int32_t amp_width;                         /* 0 or 196: the whole row; 195: without the root height (ampRootHeightObs False) */
  int32_t remove_base_rot;                   /* 0: upright start; 1: the heading and root rotation feature of remove_base_rot(q0) */
} pulse_amp_row_args_t;
int pulse_amp_obs_row(const pulse_amp_row_args_t* args, int64_t num_envs, void* stream);
int pulse_bump_counter(uint64_t* counter, uint64_t by, void* stream);
/* Timing events that stay readable when the launches around them are captured into a CUDA graph (cudaEventRecordExternal): bench.py
 * times the fused step kernel live inside a whole-rollout graph with these. */
int pulse_event_create(void** event);
int pulse_event_destroy(void* event);
int pulse_event_record(void* event, void* stream);
int pulse_event_elapsed_ms(void* start, void* stop, float* ms);

/* ------------------------------------------------------------------------------------------------
 * Per-step env reset, fused and free of host synchronisation (SURVEY row a13 / 8f-3).  Replaces, for the envs whose
 * reset_buf is set (mask mode: the `done_indices` of AMPAgent.play_steps, phc/learning/amp_agent.py:352 -> env_reset ->
 * VecTaskPythonWrapper.reset -> Humanoid.reset, humanoid.py:526-541) or for an explicit id list:
 *   HumanoidIm._reset_ref_state_init     phc/env/tasks/humanoid_im.py:921-948   (start offset / global offset / cycle counter <- 0)
 *   HumanoidAMP._reset_ref_state_init    humanoid_amp.py:468-488, _sample_ref_state humanoid_im.py:966-989
 *   MotionLibBase.sample_time_interval   phc/utils/motion_lib_base.py:411-420   (uniform draw injected or Philox)
 *   HumanoidAMP._set_env_state           humanoid_amp.py:565-597  (root 13, dof pos / vel 69, rigid bodies 24 x 13, written in place
 *                                        into the Isaac Gym views; the rigid-body write is the reference's own post-refresh hack :604-614)
 *   Humanoid._reset_env_tensors          humanoid.py:589-609      (progress / reset / terminate <- 0, contact forces <- 0, and the
 *                                        int32 actor-id list for gym.set_*_tensor_indexed, built on the device)
 *   HumanoidAMP._init_amp_obs            humanoid_amp.py:519-563  (current AMP observation + the num_steps-1 history frames at
 *                                        t - k*dt from the reference motion, no offset)
 * Two launches (ordered compaction; one warp per (env, history step)).  The observation of the reset envs follows with
 * pulse_im_step(flags = PULSE_STEP_OBS, env_ids = env_list, env_count = count).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int64_t* reset_buf;            /* [N] mask mode: envs with reset_buf != 0 are reset; cleared for them afterwards */
  const int64_t* env_ids_in;     /* list mode: explicit env ids [num_ids] (Humanoid.reset(env_ids)); NULL = mask mode */
  int64_t num_ids;
  const float* phase;            /* [N] uniform [0,1) draw per ENV (tests inject it) or NULL: Philox4x32-10(seed, env, offset) */
  uint64_t seed, offset;
  const int64_t* motion_ids;     /* [N] _sampled_motion_ids (each env keeps its clip, humanoid_im.py:966-989) */
  float* motion_start_times;     /* [N] <- sampled start time */
  float* motion_start_offset;    /* [N] <- 0 */
  float* global_offset;          /* [N,3] <- 0 */
  int32_t* cycle_counter;        /* [N] <- 0 (may be NULL) */
  int64_t* progress_buf;         /* [N] <- 0 */
  int64_t* terminate_buf;        /* [N] <- 0 (may be NULL) */
  float* root_states; int64_t root_env_stride;           /* _humanoid_root_states: env e at root_states + e*root_env_stride, 13 floats */
  float* dof_pos; float* dof_vel; int64_t dof_env_stride; int64_t dof_elem_stride;   /* Isaac Gym dof-state views (elem stride 2) */
  float* rigid_body_state; int64_t body_env_stride;      /* [N, bodies_per_env, 13]; may be NULL */
  float* contact_forces; int64_t contact_env_stride; int32_t contact_bodies;   /* [N, bodies_per_env, 3] <- 0; may be NULL */
  int32_t num_amp_steps;         /* numAMPObsSteps; 0 with amp_obs_buf NULL */
  float* amp_obs_buf;            /* [N, num_amp_steps, 196]; may be NULL */
  float dt;                      /* control dt */
  int32_t reserved;
  const int32_t* actor_ids;      /* [N] _humanoid_actor_ids (humanoid.py:590) or NULL */
  int64_t* env_list;             /* [N] out: the reset env ids, ascending (what `nonzero` returns) */
  int32_t* actor_list;           /* [N] out: actor ids of those envs (argument of gym.set_*_tensor_indexed); may be NULL */
  int32_t* count;                /* [1] out, device side: number of reset envs */
  int32_t* amp_fresh;            /* [N] optional: set to 1 for every reset env -- tells pulse_amp_obs_row to take that env's history from
                                    amp_obs_buf (the back-filled rows) at the next step */
  const uint64_t* offset_dev;    /* optional device-side counter added to `offset` (fresh draws on every CUDA-graph replay) */
} pulse_reset_args_t;
int pulse_reset_ref_state(const pulse_motionlib_t* lib, const pulse_reset_args_t* args, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Getup reset of HumanoidImGetup on the device, free of host synchronisation.  For the reset set of `base` (mask or id list), in
 * the order of HumanoidImGetup._reset_actors (phc/env/tasks/humanoid_im_getup.py:135-182):
 *   1. every reset env releases its current assignment: available_fall_states[fall_id_assignments[env]] = 0, stale or not;
 *   2. recovery envs (draw < recovery_prob and terminate_buf == 1, read before anything clears it): recovery_counter <- recovery_steps,
 *      actor state, motion id and start time kept (_reset_recovery_episode :164-166);
 *   3. fall envs (the others whose draw < fall_prob): k distinct free states, the one with the i-th smallest key to the i-th fall env in
 *      ascending env order (the distribution of randperm(available)[:k]); root / dof position / dof velocity copied from the fall pool,
 *      recovery_counter <- recovery_steps, the state marked held and assigned (_reset_fall_episode :168-182).  Where the reference
 *      asserts (fewer free states than fall envs) the surplus fall envs, the last in env order, take a reference-state episode
 *      instead and *error grows by their number;
 *   4. reference-state envs: pulse_reset_ref_state's start-time draw, MotionLib gather, scatter and AMP back-fill; recovery_counter <- 0;
 *   5. every reset env: progress / reset / terminate and its contact-force rows <- 0; the int32 actor-id list (_reset_env_tensors,
 *      humanoid.py:589-609), recovery envs included.
 * Draws: injected per env (recovery_u, fall_u: u < p succeeds) and per fall state (fall_keys, >= 0), or Philox4x32-10 on
 * (seed, index, offset + *offset_dev) of `base`: words 1 / 2 of env e's block are its recovery / fall draws, word 3 of state s's block
 * its key, so none of them meets the start-time draw (word 0 of env e's block).
 * The AMP history of fall and recovery envs depends on the state after the simulator's refresh: pulse_getup_amp_init, run after it.
 * ---------------------------------------------------------------------------------------------- */
#define PULSE_GETUP_REF 1
#define PULSE_GETUP_FALL 2
#define PULSE_GETUP_RECOVERY 3

typedef struct {
  pulse_reset_args_t base;       /* reset set, reference-state buffers, and the UNION of the reset envs in env_list / actor_list / count */
  const float* recovery_u;       /* [N] uniform draw per env, or NULL: Philox */
  const float* fall_u;           /* [N] uniform draw per env, or NULL: Philox */
  const float* fall_keys;        /* [P] non-negative key per fall state, or NULL: Philox */
  float recovery_prob;           /* _recovery_episode_prob */
  float fall_prob;               /* _fall_init_prob */
  int32_t recovery_steps;        /* _recovery_steps */
  int32_t reserved;
  int32_t* recovery_counter;     /* [N] _recovery_counter */
  int64_t* available_fall_states;/* [P] availalbe_fall_states: 0 free, 1 held */
  int64_t* fall_id_assignments;  /* [N] */
  const float* fall_root_states; int64_t fall_root_stride;       /* [P, >= 13] _fall_root_states */
  const float* fall_dof_pos; const float* fall_dof_vel;          /* [P, 69] _fall_dof_pos / _fall_dof_vel (shared strides) */
  int64_t fall_dof_env_stride; int64_t fall_dof_elem_stride;
  int64_t num_fall_states;       /* P */
  int64_t* ref_list;             /* [N] out: reference-state envs, ascending */
  int64_t* fall_list;            /* [N] out: fall envs, ascending */
  int64_t* recovery_list;        /* [N] out: recovery envs, ascending */
  int32_t* class_counts;         /* [3] out, device side: number of reference-state, fall and recovery envs */
  uint8_t* env_class;            /* [N] out, optional: PULSE_GETUP_* of every reset env (other envs untouched) */
  int32_t* error;                /* [1] in/out: += fall envs that found no free state (never cleared by the library) */
  int64_t* fall_pick;            /* [N] scratch: fall state of the i-th fall env */
  uint64_t* fall_key_scratch;    /* [P] scratch: (key, state) sort keys */
} pulse_getup_reset_args_t;
int pulse_reset_getup(const pulse_motionlib_t* lib, const pulse_getup_reset_args_t* args, int64_t num_envs, void* stream);

/* The AMP history of the fall and recovery envs of the last pulse_reset_getup, from the simulator state after the refresh
 * (humanoid_amp.py:519-533, humanoid_im_getup.py:190-196): fall envs get the current AMP observation in every row
 * (_init_amp_obs_default), recovery envs in row 0 only.  Lists and counts are pulse_reset_getup's outputs; num_envs bounds them. */
typedef struct {
  const float* body_state; int64_t body_env_stride;
  const float* dof_pos; const float* dof_vel; int64_t dof_env_stride; int64_t dof_elem_stride;
  float* amp_obs_buf;            /* [N, num_steps, 196] */
  int32_t num_steps; int32_t reserved;
  const int64_t* fall_list; const int64_t* recovery_list; const int32_t* class_counts;
} pulse_getup_amp_args_t;
int pulse_getup_amp_init(const pulse_getup_amp_args_t* args, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GAE / returns.  CommonAgent.discount_values  phc/learning/common_agent.py:493-505, mb_returns =
 * mb_advs + mb_values (amp_agent.py:427), and the first half of _calc_advs (:589-599): sums for the
 * advantage mean / unbiased std.  Inputs are [T,N] time-major as in the rl_games ExperienceBuffer;
 * outputs are written ENV-MAJOR [N,T] (swap_and_flatten01 layout) ready for minibatch slicing.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* rewards;      /* [T,N] */
  const float* values;       /* [T,N] */
  const float* next_values;  /* [T,N] already multiplied by (1-terminated), amp_agent.py:396-398 */
  const float* fdones;       /* [T,N] 0/1 */
  float gamma, tau;
  float* advantages;         /* [N,T] env-major */
  float* returns;            /* [N,T] env-major */
  double* adv_sum;           /* [2]: sum(adv), sum(adv^2) accumulated with atomics; caller zeroes; may be NULL */
} pulse_gae_args_t;
int pulse_gae(const pulse_gae_args_t* args, int32_t horizon, int64_t num_envs, void* stream);
/* advantages <- (adv - mean) / (std + 1e-8) with unbiased std from adv_sum (common_agent.py:596-597) */
int pulse_normalize_advantages(float* advantages, const double* adv_sum, int64_t count, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense layers on the tensor cores: D[M,N] = epilogue(alpha * A[M,K] . B[N,K]^T), bf16 operands (both
 * K-major: row-major with the reduction dimension contiguous), fp32 accumulation in registers (wgmma).
 * Replaces the nn.Linear + activation stacks of the policy / value / discriminator / VAE networks
 * (phc/learning/network_builder.py:105-124, amp_network_builder.py:58-249, amp_network_z_builder.py:341-467)
 * and their autograd backward: forward (A=X, B=W), dgrad (A=dY, B=W^T), wgrad (A=dY^T, B=X^T).
 * ---------------------------------------------------------------------------------------------- */
typedef uint16_t pulse_bf16_t;  /* raw bfloat16 bits */
#define PULSE_ACT_NONE 0
#define PULSE_ACT_RELU 1
#define PULSE_ACT_SILU 2

typedef struct {
  const float* bias;         /* [N] added before the activation, or NULL */
  int32_t act;               /* PULSE_ACT_* applied to (alpha*acc + bias) */
  int32_t gate_mode;         /* PULSE_ACT_RELU / PULSE_ACT_SILU: multiply by act'(gate) (backward through the activation) */
  const pulse_bf16_t* gate;  /* [M, ldg] saved tensor: ReLU -> the layer OUTPUT, SiLU -> the PRE-activation; NULL = off */
  int64_t ldg;
  float alpha;
  pulse_bf16_t* out;         /* [M, ldo] bf16 row-major, or NULL */
  int64_t ldo;
  pulse_bf16_t* out_t;       /* [N, ldot] bf16 TRANSPOSED copy (operand of the next wgrad), or NULL */
  int64_t ldot;
  float* out_f32;            /* [M, ldf] fp32 (heads, weight-gradient slabs), or NULL */
  int64_t ldf;
  int64_t split_stride;      /* floats between split-K slabs of out_f32 */
  pulse_bf16_t* preact;      /* [M, ldp] bf16 pre-activation (saved for SiLU backward), or NULL */
  int64_t ldp;
  float* colsum;             /* [N] += column sums of the final values (bias gradient of the layer whose dY this GEMM writes), or NULL */
  int32_t accumulate;        /* 1: out_f32 += result with fp32 atomics (weight gradients; caller zeroes), 0: overwrite */
  int32_t reserved;
  double* sumsq;             /* *sumsq += sum of squares of the final values over the valid [M,N] region (fp64 atomics), or NULL */
  /* ---- ABI 2: ReLU masks as bit words.  Forward: bit i of relu_mask[(col/32) * ld_rmask + row] = (pre-activation of column
   * 32*(col/32)+i of `row`) > 0, written next to the bf16 activations (2 MB instead of the 32 MB the backward pass used to re-read
   * for a 16384 x 1024 layer).  ReLU-dgrad: gate_mask in the same layout replaces `gate`: one coalesced 4-byte load per
   * (row, 32-column chunk).  Chunk-major ([ceil(N/32), ld] words, ld >= M) so that consecutive rows are consecutive words. */
  uint32_t* relu_mask; int64_t ld_rmask;
  const uint32_t* gate_mask; int64_t ld_gmask;
} pulse_gemm_epilogue_t;

#define PULSE_GEMM_A_MN 1u   /* A is given as [K, M] row-major (the reduction dimension is the ROW index) */
#define PULSE_GEMM_B_MN 2u   /* B is given as [K, N] row-major */

/* D[M,N] = epilogue(sum_k A(m,k) B(n,k)).  flags select, per operand, K-major storage (A[M,K] / B[N,K]) or MN-major
 * storage (A[K,M] / B[K,N] row-major), so activations, output gradients and weights are consumed exactly as they sit in
 * memory:  forward Y = X . W^T -> A = X, B = W, both K-major;  dgrad dX = dY . W  -> A = dY (K-major), B = W [N_out,K_in]
 * as MN-major;  wgrad dW = dY^T X -> A = dY [batch,N] MN-major, B = X [batch,K] MN-major.  No transposed copies anywhere.
 * lda / ldb in elements, multiples of 8, >= the contiguous extent (K for K-major storage); A and B 16-byte aligned.
 * split_k > 1: fp32 slabs only (slab z at out_f32 + z*split_stride); pulse_gemm_num_splits gives the number of slabs
 * actually written. */
int pulse_gemm_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, int64_t m, int64_t n, int64_t k,
                    const pulse_gemm_epilogue_t* ep, int32_t split_k, uint32_t flags, void* stream);
int pulse_gemm_num_splits(int64_t k, int32_t split_k);
/* The GEMM's shape rule alone: the output tile width (128 or 256) it picks for an m x n x k GEMM with split_k on `sms` SMs.  A launch
 * takes the wide tile only for forward / ReLU-dgrad GEMMs with a K-major A and bf16-only outputs without a pre-activation, and never
 * under PULSE_GEMM_BN=128 or PULSE_GEMM_STAGES=4.  pulse_gemm_last_launch: the kernel the last GEMM launch from the host took, as
 * out[6] = {epilogue mode (0 generic, 1 forward, 2 ReLU dgrad, 3 weight gradient, 4 general-gate dgrad), ring depth, tile width,
 * tma_out (0 staged epilogue, 1 bulk tensor stores / reductions, 2 register-resident fp32 slabs), splits, grid}; zeros before the
 * first.  pulse_gemm_last_tile_n: its tile width alone (0 before the first launch). */
int pulse_gemm_tile_n(int64_t m, int64_t n, int64_t k, int32_t split_k, int32_t sms);
int pulse_gemm_last_launch(int32_t* out);
int pulse_gemm_last_tile_n(void);

/* ------------------------------------------------------------------------------------------------
 * Element-wise / reduction kernels around the GEMMs.
 * ---------------------------------------------------------------------------------------------- */
/* RunningMeanStd.forward, eval path (phc/utils/running_mean_std.py:69-95): y = clamp((x-mean)*rstd, -5, 5),
 * written as bf16 [rows, ld_out] (columns >= cols zero-filled up to ld_out) and optionally transposed
 * bf16 [ld_out, ld_t] (operand of the first layer's wgrad).  mean / rstd: fp32 [cols] (rstd = 1/sqrt(var+eps),
 * prepared by the caller from the fp64 statistics); NULL mean = plain cast.  pad_one: value of the FIRST pad column (index cols) when
 * ld_out > cols -- 1.0 makes it the "ones" column of a bias-augmented GEMM operand (the layer's bias then sits in column `cols` of its
 * weight matrix: bias add and bias gradient ride the tensor cores), 0.0 = plain zero fill. */
int pulse_normalize_to_bf16(const float* x, int64_t ldx, int64_t rows, int64_t cols, const float* mean, const float* rstd,
                            pulse_bf16_t* out, int64_t ld_out, pulse_bf16_t* out_t, int64_t ld_t, float pad_one, void* stream);

/* Batch moments for RunningMeanStd's training-mode update (:96-107): per-column sum and sum of squares of
 * fp32 x [rows, cols] accumulated in fp64 into sums[2*cols] (caller zeroes). */
int pulse_column_moments(const float* x, int64_t ldx, int64_t rows, int64_t cols, double* sums, void* stream);

/* pulse_normalize_to_bf16 + pulse_column_moments in ONE pass over x: RunningMeanStd.forward in training mode
 * (phc/utils/running_mean_std.py:91-107) normalises with the statistics from before the batch and merges the
 * batch afterwards, so both read the same rows.  out [rows, ld_out] (padding columns zeroed), sums[2*cols] += . */
int pulse_normalize_moments(const float* x, int64_t ldx, int64_t rows, int64_t cols, const float* mean, const float* rstd,
                            pulse_bf16_t* out, int64_t ld_out, double* sums, float pad_one, void* stream);

/* The same normalisation for an observation [self | task] that feeds two bias-augmented first layers (the amp_sept network:
 * a task encoder whose output joins the self observation), in ONE pass over x [rows, cols]:
 *   p [rows, ldp] = [columns 0..p_off-1 untouched (the encoder output goes there) | self (self_cols) | 1 | 0 ...]
 *   t [rows, ldt] = [task (cols - self_cols) | 1 | 0 ...]
 * sums[2*cols] += the batch moments of all cols columns when sums != NULL (training mode); NULL = normalise only.
 * cols, self_cols, p_off, ldp, ldt and ldx even; x, mean, rstd 8-byte and p, t 4-byte aligned. */
int pulse_normalize_split(const float* x, int64_t ldx, int64_t rows, int64_t cols, int64_t self_cols, const float* mean, const float* rstd,
                          pulse_bf16_t* p, int64_t ldp, int64_t p_off, pulse_bf16_t* t, int64_t ldt, double* sums, void* stream);

/* RunningMeanStd._update_mean_var_count_from_moments (:54-66) on the device: merges the batch sums of
 * pulse_column_moments (n rows) into the fp64 running mean / var / count and refreshes the fp32 mean / rstd
 * vectors pulse_normalize_to_bf16 reads, then zeroes `sums` for the next batch.  One launch, no host round trip. */
int pulse_rms_merge(double* sums, int64_t n, int32_t size, double* mean, double* var, double* count, float eps,
                    float* mean_f32, float* rstd_f32, void* stream);

/* Single-output head (the critic's `value` Linear, network_builder.py:171; the discriminator's `_disc_logits`,
 * amp_network_builder.py:245-249): out[m] = h[m,:] . w + bias.  h bf16 [rows, k] (row stride ldh), w bf16 [k]. */
int pulse_head1_forward(const pulse_bf16_t* h, int64_t ldh, int64_t rows, int32_t k, const pulse_bf16_t* w, const float* bias, float* out,
                        int64_t ldo, void* stream);

/* Backward of that head through the ReLU below it, ONE pass over h:  dh[m,j] = dv[m] w[j] (h[m,j] > 0) (bf16, may be
 * NULL);  dw[j] += sum_m dv[m] h[m,j];  db += sum_m dv[m];  dbias_prev[j] += sum_m dh[m,j] (bias gradient of the layer
 * that produced h; may be NULL).  k <= 2048, multiple of 8.  partials: fp32 scratch of PULSE_HEAD1_MAX_CTAS * (2k + 1) floats
 * (per-CTA sums, added in CTA order: the result does not depend on scheduling). */
#define PULSE_HEAD1_MAX_CTAS 264
int pulse_head1_backward(const pulse_bf16_t* h, int64_t ldh, int64_t rows, int32_t k, const pulse_bf16_t* dv, int64_t ld_dv,
                         const pulse_bf16_t* w, pulse_bf16_t* dh, int64_t ld_dh, float* dw, float* db, float* dbias_prev, float* partials,
                         void* stream);

/* out[r, c] += sum_{s < n} x[s * stride_n + r * ld + c], the n terms added in the order s = 0, 1, ... (split-K slabs, partial sums):
 * a reduction that gives the same bits on every run.  ld / ldo are ignored when rows == 1. */
int pulse_ordered_sum_add(const float* x, int64_t n, int64_t stride_n, int64_t rows, int64_t cols, int64_t ld, float* out, int64_t ldo,
                          void* stream);

/* Gaussian policy head (rl_games ModelA2CContinuousLogStd, fixed sigma: im.yaml:21-25):
 * actions = mu + exp(logstd)*eps;  neglogp = 0.5*sum(((a-mu)/sigma)^2) + 0.5*A*log(2*pi) + sum(logstd). */
int pulse_gaussian_sample(const float* mu, int64_t ld_mu, const float* eps, const float* logstd, int64_t rows, int32_t num_actions,
                          float* actions, float* neglogp, void* stream);

/* PPO actor / critic / bound losses and their gradients w.r.t. the network outputs, one pass
 * (common_agent.py:512-520, :564-587; amp_agent.py:691-710; torch_ext.policy_kl):
 *   a = max(-A r, -A clip(r, 1-e, 1+e)), r = exp(old_neglogp - neglogp);  c = (ret - v)^2;
 *   b = sum(clamp_min(mu-1,0)^2 + clamp_max(mu+1,0)^2);  loss = mean(a) + critic_coef*mean(c) + bounds_coef*mean(b).
 * Outputs: dmu bf16 [rows, ld_dmu] (+ transposed [A_pad, ld_t]), dvalue bf16 [rows, ld_dv] (+ transposed),
 * stats[0..5] fp64 accumulators: sum a, sum c, sum b, sum kl, clipped count, sum neglogp (caller zeroes).  1 <= num_actions <= 256. */
typedef struct {
  const float* mu; int64_t ld_mu;       /* [rows, A] network output */
  const float* value; int64_t ld_value; /* [rows, 1] */
  const float* actions;                 /* [rows, A] contiguous */
  const float* old_neglogp;             /* [rows] */
  const float* advantages;              /* [rows] */
  const float* returns;                 /* [rows] (already value-normalised) */
  const float* old_mu;                  /* [rows, A] contiguous, for the KL statistic; may be NULL */
  const float* logstd;                  /* [A] */
  int32_t num_actions;
  float e_clip, critic_coef, bounds_coef;
  pulse_bf16_t* dmu; int64_t ld_dmu; pulse_bf16_t* dmu_t; int64_t ld_dmu_t;
  pulse_bf16_t* dvalue; int64_t ld_dv; pulse_bf16_t* dvalue_t; int64_t ld_dv_t;
  double* stats;
} pulse_ppo_loss_args_t;
int pulse_ppo_loss(const pulse_ppo_loss_args_t* args, int64_t rows, void* stream);

/* AMP discriminator loss pieces (AMPAgent._disc_loss, phc/learning/amp_agent.py:895-952):
 *  - prediction loss 0.5*(BCE(agent U replay, 0) + BCE(demo, 1)) and its gradient w.r.t. the logits
 *    (rows [0,n_agent) agent/replay, rows [n_agent, n_agent+n_demo) demo), scaled by `scale` (= disc_coef);
 *    stats[0..3] += sum softplus(l) agent, sum softplus(-l) demo, #agent l<0, #demo l>0 (accuracies, :954-959);
 *  - pulse_relu_mask_scale: out = (h > 0) * w, the first factor of the ANALYTIC input gradient of the ReLU
 *    discriminator used for the gradient penalty (:910-929) instead of autograd's double backward;
 *  - pulse_axpy: y += a*x (logit regulariser :905-908 and weight decay :932-937 gradients, 2*coef*w). */
int pulse_disc_loss(const float* logits, int64_t ld, int64_t n_agent, int64_t n_demo, float scale, pulse_bf16_t* dlogit, int64_t ld_d,
                    double* stats, void* stream);
int pulse_relu_mask_scale(const pulse_bf16_t* h, int64_t ldh, int64_t rows, int64_t cols, const float* w, pulse_bf16_t* out, int64_t ldo,
                          void* stream);
int pulse_axpy(float a, const float* x, float* y, int64_t count, void* stream);
/* Weight decay / logit regulariser gradients + the sums of squares of the logged terms for up to four weight blocks in one launch
 * (AMPAgent._disc_loss, amp_agent.py:905-908, :932-937): g[r,c] += coef * w[r,c] for c < cols of a [rows, ld] matrix; *sumsq (and
 * *sumsq2) += sum w^2 in fp64.  g / sumsq / sumsq2 may be NULL. */
typedef struct {
  const float* w; float* g; int64_t rows, cols, ld; float coef; int32_t reserved; double* sumsq; double* sumsq2;
} pulse_weight_block_t;
typedef struct { pulse_weight_block_t block[4]; int32_t count; int32_t reserved; } pulse_weight_reg_t;
int pulse_weight_reg(const pulse_weight_reg_t* desc, void* stream);

/* out[c] (+)= sum over rows of bf16 x[rows, ldx] (bias gradients). */
int pulse_column_sum_bf16(const pulse_bf16_t* x, int64_t ldx, int64_t rows, int64_t cols, float* out, void* stream);
/* dst[i] = sum_s slabs[s*slab_stride + i]  (split-K weight-gradient slabs -> flat gradient buffer) */
int pulse_reduce_slabs(const float* slabs, int64_t slab_stride, int32_t num_slabs, int64_t count, float* dst, void* stream);
/* sumsq[0] += sum(x^2) in fp64 (global gradient norm; caller zeroes) */
int pulse_sum_squares(const float* x, int64_t count, double* sumsq, void* stream);
/* clip_grad_norm_(max_norm) + Adam step over one flat parameter buffer (amp_agent.py:725-750; torch.optim.Adam
 * defaults beta 0.9/0.999): scale = min(1, max_norm/(sqrt(sumsq)+1e-6)) read on the device, no host sync. */
/* `step` is a DEVICE counter (int32[1]) incremented by this call, so the launch sequence is CUDA-graph replayable.
 * params_bf16 (optional, same flat layout): bf16 copy of the updated parameters = the GEMM operands. */
#define PULSE_ADAM_ZERO_GRADS 1u      /* the kernel zeroes every gradient it has consumed (the next minibatch accumulates from zero) */
#define PULSE_ADAM_SELF_CONTAINED 2u  /* no bump / memset launches: this launch is step *step + 1; its last block stores the new step and
                                         re-zeroes *grad_sumsq (block_counter: one zero-initialised uint32 owned by the optimizer) */
int pulse_adam_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, int64_t count, double* grad_sumsq,
                    float max_norm, float lr, float beta1, float beta2, float eps, int32_t* step, pulse_bf16_t* params_bf16, uint32_t flags,
                    uint32_t* block_counter, void* stream);
/* Multi-GPU optimizer step over NVLink peer memory (csrc/peer_adam.cu): the reference's Horovod gradient averaging
 * (hvd.DistributedOptimizer, amp_agent.py:735-742) + clip_grad_norm_ + torch.optim.Adam (amp_agent.py:725-750) as ONE kernel per rank --
 * reduce-scatter of the flat gradient buffers by peer loads (or multimem.ld_reduce), exchange of the slice norms, Adam on the rank's
 * slice (sharded moments), push of the new fp32 masters + bf16 operands into every rank's buffers (peer stores or multimem.st), clearing
 * of the gradients.  Replaces pulse_sum_squares + pulse_adam_step + the NCCL all-reduce when the ranks' buffers are peer-mapped.
 *   grads / params / params_bf16 / signals [p]: rank p's buffer as mapped into THIS process ([rank] = the local one).  A signal block
 *   is PULSE_PEER_SIGNAL_BYTES of zero-initialised memory: uint32 flags[3][PULSE_PEER_MAX] then double norms[PULSE_PEER_MAX].
 *   mc_*: multicast aliases of the same buffers (NVLS), or NULL.  exp_avg / exp_avg_sq: local, full size; only this rank's slice
 *   [rank * ceil(count/4/world) * 4, ...) is read or written.  step: device Adam step counter (incremented).  epoch: device uint32[1]
 *   call counter, zero-initialised, same value on every rank.  cta_partials: double[PULSE_PEER_MAX_GRID]; grid_bar: uint64[1] zero-
 *   initialised; grid: CTAs (0 = one per SM) -- must not change between calls that share grid_bar.
 * Every rank must make the call (it waits for its peers, bounded by timeout_ms, then the launch fails); count is a multiple of 4. */
#define PULSE_PEER_MAX 8
#define PULSE_PEER_MAX_GRID 256
#define PULSE_PEER_SIGNAL_BYTES (3 * PULSE_PEER_MAX * 4 + PULSE_PEER_MAX * 8)
typedef struct {
  int32_t rank, world;
  float* grads[PULSE_PEER_MAX];
  float* params[PULSE_PEER_MAX];
  pulse_bf16_t* params_bf16[PULSE_PEER_MAX];
  uint32_t* signals[PULSE_PEER_MAX];
  const float* mc_grads; float* mc_params; pulse_bf16_t* mc_params_bf16;
  float* exp_avg; float* exp_avg_sq;
  int64_t count;
  float max_norm, lr, beta1, beta2, eps;
  int32_t grid;
  uint32_t timeout_ms;                     /* bound of every wait on a peer (0 = 30 min: ranks drift apart around rank-0-only work) */
  uint32_t reserved;
  int32_t* step;
  uint32_t* epoch;
  double* cta_partials;
  unsigned long long* grid_bar;
} pulse_peer_adam_args_t;
int pulse_peer_reduce_adam(const pulse_peer_adam_args_t* args, void* stream);

/* refresh the bf16 operand copies of one weight matrix W fp32 [n, k] (contiguous):
 *   w_bf16 [n, ld_k] (K-major, forward / wgrad-free) and wt_bf16 [k, ld_n] (transposed, dgrad operand); pads zeroed. */
int pulse_refresh_weight_bf16(const float* w, int64_t n, int64_t k, pulse_bf16_t* w_bf16, int64_t ld_k, pulse_bf16_t* wt_bf16,
                              int64_t ld_n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * PULSE VAE distillation (SURVEY K17-K19), Z-task decode (K20), reach task (K21), PD targets (K22).
 * The dense layers run on pulse_gemm_bf16; these are the row-wise pieces between them.
 * ---------------------------------------------------------------------------------------------- */
/* y = (x - mean) * rstd, optionally clamped to [-clamp, clamp] (clamp <= 0: no clamp -- HumanoidZ.compute_z_actions feeds the
 * prior the UNCLAMPED normalised self observation, humanoid_z.py:87 vs :147), written as bf16 into out[rows, 0:cols];
 * columns [cols, zero_to) of each out row are zero-filled, nothing beyond is touched (out may be a column window of a wider
 * operand buffer).  mean/rstd NULL = plain cast. */
int pulse_normalize_cols(const float* x, int64_t ldx, int64_t rows, int64_t cols, const float* mean, const float* rstd, float clamp,
                         pulse_bf16_t* out, int64_t ld_out, int64_t zero_to, void* stream);
/* dst1[r, 0:cols] = dst2[r, 0:cols] = src[r, 0:cols] (bf16; dst2 may be NULL): the normalised self-observation columns of
 * the encoder input feed the prior MLP and the decoder input window (amp_network_z_builder.py:229, :443-445). */
int pulse_copy_cols_bf16(const pulse_bf16_t* src, int64_t ld_src, int64_t rows, int64_t cols, pulse_bf16_t* dst1, int64_t ld1,
                         pulse_bf16_t* dst2, int64_t ld2, void* stream);

/* Latent sample (form_embedding / reparameterize, amp_network_z_builder.py:79-121, :243-246).  head fp32 [rows, >= 2*latent]:
 * columns [0, latent) = mu, [latent, 2*latent) = raw log-variance (clamped to [clamp_lo, clamp_hi] when clamp != 0).
 *   mode PULSE_Z_SAMPLE: z = mu + exp(0.5*logvar)*noise;  PULSE_Z_MEAN: z = mu (flags.test, :94-95);
 *   PULSE_Z_RESIDUAL:    z = mu + noise  (HumanoidZ.compute_z_actions: prior_mu + action_z, humanoid_z.py:104-107).
 * z is written as bf16 into z_bf16[rows, 0:latent] (the decoder input window) and/or fp32 z_f32[rows, latent]. */
#define PULSE_Z_SAMPLE 0
#define PULSE_Z_MEAN 1
#define PULSE_Z_RESIDUAL 2
int pulse_vae_reparam(const float* head, int64_t ld_head, const float* noise, int64_t ld_noise, int64_t rows, int32_t latent,
                      int32_t mode, int32_t clamp, float clamp_lo, float clamp_hi, pulse_bf16_t* z_bf16, int64_t ld_z, float* z_f32,
                      int64_t ld_zf, void* stream);
/* PULSE_Z_SAMPLE with the noise drawn in the kernel (the distillation rollout, amp_network_z_builder.py:82-95 in eval mode):
 * z = mu + exp(0.5*clamp(logvar, clamp_lo, clamp_hi))*eps written as bf16 into z_bf16[rows, 0:latent], latent <= 32.
 * eps ~ N(0,1) from Philox4x32-10 keyed (seed, row*64 + j/2) with offset (*offset_dev if not NULL) + step; the two words of one call
 * give the Box-Muller pair (j, j+1).  noise_out fp32 [rows, latent] (or NULL) receives eps. */
int pulse_vae_reparam_philox(const float* head, int64_t ld_head, int64_t rows, int32_t latent, int32_t clamp, float clamp_lo,
                             float clamp_hi, uint64_t seed, const uint64_t* offset_dev, uint64_t step, pulse_bf16_t* z_bf16,
                             int64_t ld_z, float* noise_out, int64_t ld_noise, void* stream);

/* kin_action_loss = mean_rows ||pred - gt||_2 (amp_agent.py:782): stats[0] += sum of row norms (fp64; caller zeroes);
 * dpred bf16 [rows, ld_d] = (pred - gt) / (||pred - gt|| * rows) (0 where the norm is 0, as torch.norm's backward), columns
 * [num_actions, zero_to) zero-filled. */
int pulse_vae_action_loss(const float* pred, int64_t ld_pred, const float* gt, int64_t ld_gt, int64_t rows, int32_t num_actions,
                          pulse_bf16_t* dpred, int64_t ld_d, int64_t zero_to, double* stats, void* stream);

/* Latent-space terms of AMPAgent._optimize_kin (amp_agent.py:784-816) and their gradients w.r.t. the encoder / prior heads,
 * one warp per row (latent <= 32):
 *   KLD  = mean_rows kl_multi(q || p)                                   (loss_functions.py:3-11)      * kld_coef
 *   AR1  = mean over (rows/horizon)*(horizon-1) pairs of ||mu[t+1] - phi mu[t]||, pairs masked where the progress counter is
 *          not consecutive or either step has progress <= 2 (:792-808)                                   * ar1_coef
 *   REGU = 0.001*(mean pm^2 + mean qm^2 + mean pv^2 + mean qv^2) (:810-814)                              * regu_coef
 * plus the reparameterisation path of dz = dLoss/dz (from the decoder's input gradient):  dmu += dz,
 * dlogvar += dz * 0.5*exp(0.5*logvar)*noise; clamp gates (gradient passes where lo <= raw <= hi).
 * Rows are env-major [rows/horizon, horizon] (amp_datasets.py:54-79).  progress NULL or ar1_coef == 0: no AR(1) term.
 * stats (fp64, caller zeroes): [0] sum KL rows, [1] sum AR1 pair norms, [2] sum pm^2, [3] sum qm^2, [4] sum pv^2, [5] sum qv^2. */
typedef struct {
  const float* enc_head; int64_t ld_enc;       /* [rows, >= 2*latent]: mu | raw logvar of the posterior */
  const float* prior_head; int64_t ld_prior;   /* [rows, >= 2*latent]: mu | raw logvar of the prior */
  const float* noise; int64_t ld_noise;        /* [rows, latent] */
  const float* dz; int64_t ld_dz;              /* [rows, latent] fp32, or NULL */
  const int64_t* progress;                     /* [rows] progress_buf recorded with the sample, or NULL */
  int32_t latent, horizon, clamp, reserved;
  float clamp_lo, clamp_hi, kld_coef, ar1_coef, regu_coef, phi;
  pulse_bf16_t* d_enc_head; int64_t ld_de;     /* [rows, 2*latent] gradient w.r.t. enc_head */
  pulse_bf16_t* d_prior_head; int64_t ld_dp;   /* [rows, 2*latent] gradient w.r.t. prior_head */
  double* stats;
} pulse_vae_latent_args_t;
int pulse_vae_latent_loss(const pulse_vae_latent_args_t* args, int64_t rows, void* stream);

/* Distillation teacher output (HumanoidImDistill.step, humanoid_im_distill.py:193-198): out[r, :] = sum_k act(w[r, k]) *
 * acts[k][r, :], acts = num_prim column outputs fp32 at acts + k*prim_stride, w = raw composer head [rows, num_prim];
 * act = PULSE_ACT_SILU for the composer rebuilt by load_mcp_mlp (network_loader.py:37-39). */
int pulse_pnn_compose(const float* acts, int64_t prim_stride, int64_t ld_a, const float* w, int64_t ld_w, int32_t act, int64_t rows,
                      int32_t num_actions, int32_t num_prim, float* out, int64_t ld_out, void* stream);

/* Humanoid._action_to_pd_targets + the freeze_hand / freeze_toe zeroing of pre_physics_step (humanoid.py:1222-1247,1392-1394):
 * out = freeze[d] ? 0 : offset[d] + scale[d]*action[r, d].  freeze: uint8 [dofs] or NULL. */
int pulse_pd_targets(const float* action, int64_t ld_a, const float* offset, const float* scale, const uint8_t* freeze, int64_t rows,
                     int32_t dofs, float* out, int64_t ld_out, void* stream);

/* Pre-physics step of the distillation rollout (HumanoidImDistillGetup: pre_physics_step, then _update_recovery_count,
 * humanoid_im_getup.py:76-80) in one launch over `rows` envs:
 *   pd_out[r, d]       = freeze[d] ? 0 : offset[d] + scale[d]*mus[r, d]     (pulse_pd_targets' arithmetic)
 *   kin_progress[r]    = progress_buf[r]                                   (the progress record, humanoid_im_distill.py:205)
 *   recovery_counter[r] = max(recovery_counter[r] - 1, 0)
 * mus, pd_out and kin_progress are addressed through their row strides (experience-buffer slices). */
int pulse_distill_pre_physics(const float* mus, int64_t ld_mus, const float* pd_offset, const float* pd_scale, const uint8_t* freeze,
                              int64_t rows, int32_t dofs, float* pd_out, int64_t ld_pd, const int64_t* progress_buf,
                              int64_t* kin_progress, int64_t ld_progress, int32_t* recovery_counter, void* stream);

/* HumanoidReach._update_task / _reset_task (humanoid_reach.py:126-147) with the uniform draws supplied by the caller:
 * where progress >= tar_change_steps: tar_pos = (dist_max*(2u-1), dist_max*(2v-1), h_min + (h_max-h_min)*w),
 * tar_change_steps = progress + steps.  rand01 fp32 [n, 3], steps int64 [n]. */
int pulse_reach_update_task(const int64_t* progress, int64_t* tar_change_steps, float* tar_pos, const float* rand01, const int64_t* steps,
                            float dist_max, float h_min, float h_max, int64_t num_envs, void* stream);

/* HumanoidReach post-physics step (humanoid_reach.py:149-166, :224-250; humanoid.py:1573-1608, :1675-1731), one warp per env:
 * reward = exp(-4 ||tar - reach_body||^2); reset / terminate = compute_humanoid_reset (contact force > 0.1 on a non-contact body
 * AND a non-contact body below its termination height, progress > 1; or progress >= max_episode_length - 1);
 * obs[env] = [self observation 358 | heading-frame target offset 3]. */
typedef struct {
  const float* body_state; int64_t body_env_stride;       /* [N, >=24, 13] pos quat(xyzw) linvel angvel */
  const float* contact_forces; int64_t contact_env_stride; /* [N, >=24, 3] or NULL (no early termination) */
  const float* termination_heights;                        /* [24] */
  const float* tar_pos;                                    /* [N, 3] */
  const int64_t* progress_buf;                             /* [N] */
  uint32_t contact_body_mask;                              /* bit j: body j may touch the ground (contact_bodies) */
  int32_t reach_body_id;
  int32_t enable_early_termination, reserved;
  int64_t max_episode_length;
  float* obs_buf; int64_t obs_stride;                      /* [N, 361] */
  float* rew_buf;                                          /* [N] */
  int64_t* reset_buf; int64_t* terminate_buf;              /* [N] */
} pulse_reach_step_args_t;
#define PULSE_REACH_OBS 361
int pulse_reach_step(const pulse_reach_step_args_t* args, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Post-physics step of the downstream latent-space tasks HumanoidSpeedZ / HumanoidStrikeZ (SURVEY 8f-4), siblings of pulse_reach_step:
 * self observation (humanoid.py:1675-1731) + task observation + reward + reset in one launch.
 *   PULSE_ZTASK_SPEED   compute_speed_observations / compute_speed_reward (phc/env/tasks/humanoid_speed.py:310-343), power term
 *                       (:215-222; dof_force NULL = off), compute_humanoid_reset (humanoid.py:1573-1608).  obs 358 + 3.
 *   PULSE_ZTASK_STRIKE  compute_strike_observations / compute_strike_reward (humanoid_strike.py:270-328), the strike variant of
 *                       compute_humanoid_reset (:330-375).  obs 358 + 15.
 * prev_root_pos [N,3] = root position before the physics step (pre_physics_step, humanoid_speed.py:73-76).  Not covered: the
 * power_usage_reward terms (:224-240, humanoid_strike.py:186-198), the input-noise suffix (humanoid_speed.py:194-195).
 * ---------------------------------------------------------------------------------------------- */
#define PULSE_ZTASK_SPEED 1
#define PULSE_ZTASK_STRIKE 2
#define PULSE_SPEED_OBS 361
#define PULSE_STRIKE_OBS 373
typedef struct {
  int32_t kind, enable_early_termination;
  const float* body_state; int64_t body_env_stride;
  const float* contact_forces; int64_t contact_env_stride;      /* [N, B, 3] view or NULL */
  const float* termination_heights;                              /* [24] */
  uint32_t contact_body_mask;                                    /* bodies allowed to touch the ground (_contact_body_ids) */
  uint32_t strike_body_mask;                                     /* strike: bodies allowed to hit the target (_strike_body_ids) */
  const int64_t* progress_buf; int64_t max_episode_length;
  const float* prev_root_pos; float dt; float power_coefficient;
  const float* tar_speed;                                        /* speed: [N] */
  const float* target_states; int64_t target_env_stride;         /* strike: [N, 13] view of the target actor's root state */
  const float* tar_contact_forces; int64_t tar_contact_env_stride;   /* strike: [N, 3] view */
  const float* dof_force; int64_t dof_force_stride;              /* speed power term: [N, 69] */
  const float* dof_vel; int64_t dof_env_stride, dof_elem_stride;
  float* obs_buf; int64_t obs_stride; float* rew_buf; float* reward_raw; int64_t raw_stride;
  int64_t* reset_buf; int64_t* terminate_buf;
} pulse_ztask_step_args_t;
int pulse_ztask_step(const pulse_ztask_step_args_t* args, int64_t num_envs, void* stream);

/* The observation-only part of pulse_reach_step / pulse_ztask_step over env_list[0 .. *count) (device-side count, num_envs bounds it):
 * _compute_observations(env_ids) of the reset envs.  The same per-env code as the step kernels writes the same rows bit for bit; no
 * reward, reset or terminate word and no other row is written.  The argument structs are the step's; only the observation inputs
 * (body_state, tar_pos / tar_speed / target_states, obs_buf) are read. */
int pulse_reach_obs_list(const pulse_reach_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs, void* stream);
int pulse_ztask_obs_list(const pulse_ztask_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Reference-state reset of the latent-space tasks HumanoidReach(Z) / HumanoidSpeed(Z) / HumanoidStrike(Z), free of host
 * synchronisation: HumanoidAMPTask._reset_envs for StateInit.Random / Start and humanoid_type "smpl", without its observation and
 * _reset_task (those follow: the task's observation over env_list, then pulse_ztask_reset_task).  For the reset set (reset_buf mask
 * or env id list), two launches:
 *   1. ordered compaction into env_list / actor_list / tar_actor_list and a device-side count;
 *   2. one warp per (reset env, AMP history step k):
 *      - clip: sample_motions (motion_lib_base.py:395-398), a new clip per reset env: injected, or an inverse-CDF search of a
 *        Philox uniform over sampling_cdf (zero-weight clips are never drawn);
 *      - start time: sample_time_interval (:411-420) for PULSE_ZINIT_RANDOM, 0 for PULSE_ZINIT_START;
 *      - get_motion_state without offset, then the SMPL ground fix of _get_fixed_smpl_state_from_motionlib (humanoid_amp.py:382-430):
 *        d = (floor[f0] + root_z) - 0.02 with f0 the unblended frame, root_z -= d and every body z -= d;
 *      - pose_mode: AS_IS; ROOT_XY_ZERO (humanoid_reach.py:46-48, humanoid_strike.py:147-150: root xy <- 0, bodies keep theirs);
 *        FACE_X (humanoid_speed.py:251-270: the heading inverse of root_rot, or of remove_base_rot(root_rot) when !upright, rotates
 *        root_rot, the bodies about the root, body rotations, root velocity, root angular velocity and body velocities; body angular
 *        velocities and dofs stay);
 *      - _set_env_state (humanoid_amp.py:565-597) into the root, dof and rigid-body views, _sampled_motion_ids / _motion_start_times
 *        (:484-485), and _reset_env_tensors (humanoid.py:589-609): progress / reset / terminate and contact forces <- 0;
 *      - strike (target_states != NULL): _reset_target (humanoid_strike.py:124-145) around the new root xy;
 *      - AMP history (humanoid_amp.py:519-563): row 0 from the rigid bodies and dofs just written (what _compute_amp_observations
 *        reads after the _reset_rb_* restore), rows k >= 1 from the UNADJUSTED motion at t0 - k*dt.  amp_width 196 is the layout of
 *        pulse_reset_ref_state, 195 the same without the root height (ampRootHeightObs False, :305-306).
 * Draws: injected per ENV, or Philox4x32-10 on (seed, index, offset + *offset_dev), one word per draw:
 *   index e            x: start-time phase (the word pulse_reset_ref_state uses)   y: clip   z: strike near   w: strike distance
 *   index e + 2^32     x: strike bearing   y: strike yaw
 *   index e + 2^33     pulse_ztask_reset_task: x, y, z task uniforms, w change steps
 *   index e + 3 * 2^32 pulse_ztask_pre_physics (_update_task of the rollout): x, y, z task uniforms, w change steps
 *   index e + 4 * 2^32 pulse_traj_reset_list: counter PULSE_TRAJ_VERTS * (offset + *offset_dev) + k, k <= PULSE_TRAJ_VERTS - 1
 *                      (the pedestrian terrain task's waypoints; block k < S: segment k, block S: heading and speed)
 * The AMP demo and replay rings (pulse_amp_demo_fetch, pulse_amp_replay_store, pulse_amp_ring_sample) key their draws by the ring's own
 * seed, one index plane per draw (PULSE_PLANE_* below, i.e. index i + plane * 2^32), counter = the ring's draw or permutation counter:
 *   index i + 5 * 2^32 x: demo clip of fetched row i (inverse CDF)       counter ctr[PULSE_RING_DRAWS]
 *   index i + 6 * 2^32 x: demo start-time phase of fetched row i         counter ctr[PULSE_RING_DRAWS]
 *   index r + 7 * 2^32 x: replay keep mask of stored row r (u < p)       counter ctr[PULSE_RING_DRAWS]
 *   index 8 * 2^32     x, y, z, w: Feistel round keys of the subset      counter ctr[PULSE_RING_DRAWS]
 *   index 9 * 2^32     x, y, z, w: Feistel round keys of the sampling permutation   counter ctr[PULSE_RING_PERM_KEY]
 * pulse_reset_terrain reads index e as above, with word z as the spawn location (w unused).
 * pulse_policy_post keys its action noise by the policy's own seed, counter *rng_offset + rng_step, one block per action pair
 * p = k / 2 of row r (words x, y: actions 2p, 2p + 1 by Box-Muller; z, w unused):
 *   num_actions <= 128        index r * 64 + p    (p < 64)
 *   128 < num_actions <= 256  index r * 128 + p   (p < 128; the SMPL-X dof-space policy, 153 actions)
 * so the blocks of two rows never overlap at either width.
 * ---------------------------------------------------------------------------------------------- */
#define PULSE_ZTASK_REACH 3
#define PULSE_ZPOSE_AS_IS 0
#define PULSE_ZPOSE_ROOT_XY_ZERO 1
#define PULSE_ZPOSE_FACE_X 2
#define PULSE_ZINIT_RANDOM 0
#define PULSE_ZINIT_START 1
#define PULSE_AMP_OBS_NO_HEIGHT 195

typedef struct {
  int64_t* reset_buf;            /* [N] mask mode: envs with reset_buf != 0 are reset; cleared for them */
  const int64_t* env_ids_in;     /* list mode: ascending env ids [num_ids] (an id outside [0, N) or not above its predecessor is
                                    skipped); NULL = mask mode */
  int64_t num_ids;
  const int64_t* motion_ids_in;  /* [N] injected clip per env, or NULL: Philox + inverse CDF */
  const float* motion_u;         /* [N] injected clip uniform per env (inverse CDF), or NULL; ignored with motion_ids_in */
  const float* phase;            /* [N] injected start-time uniform per env, or NULL: Philox */
  const float* strike_u;         /* [N, 4] injected strike uniforms (near, distance, bearing, yaw) per env, or NULL: Philox */
  const float* sampling_cdf;     /* [num_motions] inclusive fp32 prefix sum of _sampling_batch_prob; required without motion_ids_in */
  uint64_t seed, offset;
  const uint64_t* offset_dev;    /* optional device-side counter added to `offset` */
  const float* floor;            /* [floor_len >= total_frames] per-frame min vertex z - root joint z at zero translation */
  int64_t floor_len;
  int32_t pose_mode;             /* PULSE_ZPOSE_* */
  int32_t upright;               /* _has_upright_start (FACE_X heading and the AMP rotation features) */
  int32_t state_init;            /* PULSE_ZINIT_* */
  int32_t amp_width;             /* 196 or 195 (SMPL-X: 466 or 465) */
  int32_t num_amp_steps;         /* numAMPObsSteps; 0 with amp_obs_buf NULL */
  float dt;                      /* control dt */
  float* amp_obs_buf;            /* [N, num_amp_steps, amp_width] or NULL */
  int64_t* sampled_motion_ids;   /* [N] <- clip */
  float* motion_start_times;     /* [N] <- start time */
  int64_t* progress_buf;         /* [N] <- 0 */
  int64_t* terminate_buf;        /* [N] <- 0 (may be NULL) */
  float* root_states; int64_t root_env_stride;
  float* dof_pos; float* dof_vel; int64_t dof_env_stride; int64_t dof_elem_stride;
  float* rigid_body_state; int64_t body_env_stride;      /* [N, bodies_per_env, 13], required */
  float* contact_forces; int64_t contact_env_stride; int32_t contact_bodies;   /* <- 0; may be NULL */
  int32_t reserved;
  float* target_states; int64_t target_env_stride;       /* strike: [N, 13] view of the target actor's root state; NULL otherwise */
  float near_prob, near_dist, tar_dist_min, tar_dist_max;
  const int32_t* actor_ids;      /* [N] _humanoid_actor_ids or NULL (env id) */
  const int32_t* tar_actor_ids;  /* [N] _tar_actor_ids or NULL (env id) */
  int64_t* env_list;             /* [N] out: the reset env ids, ascending */
  int32_t* actor_list;           /* [N] out, optional */
  int32_t* tar_actor_list;       /* [N] out, optional */
  int32_t* count;                /* [1] out, device side */
  int32_t* amp_fresh;            /* [N] optional: set to 1 for every reset env -- pulse_amp_obs_row then takes that env's history from
                                    amp_obs_buf (the back-filled rows) at the next step; requires amp_obs_buf */
} pulse_ztask_reset_args_t;
int pulse_reset_ztask(const pulse_motionlib_t* lib, const pulse_ztask_reset_args_t* args, int64_t num_envs, void* stream);

/* _reset_task of the reach and speed tasks over the env list of pulse_reset_ztask (run after the observation, as the reference does),
 * draws injected per env or Philox words of index e + 2^33:
 *   PULSE_ZTASK_REACH  humanoid_reach.py:134-146  tar_pos = (dist_max (2u - 1), dist_max (2v - 1), height_scale w + height_min)
 *   PULSE_ZTASK_SPEED  humanoid_speed.py:166-175  tar_speed = speed_scale u + speed_min
 * and change_steps = progress + randint(steps_min, steps_max); from a Philox word w, steps_min + (w (steps_max - steps_min)) >> 32. */
typedef struct {
  int32_t kind; int32_t reserved;
  const int64_t* env_list; const int32_t* count;
  const float* rand;             /* injected: reach [N, 3], speed [N]; or NULL: Philox */
  const int64_t* steps_in;       /* injected randint results [N], or NULL: Philox */
  uint64_t seed, offset;
  const uint64_t* offset_dev;
  const int64_t* progress_buf;
  int64_t* change_steps;         /* _tar_change_steps / _speed_change_steps */
  float* tar_pos;                /* reach [N, 3] */
  float* tar_speed;              /* speed [N] */
  float dist_max, height_scale, height_min, speed_scale, speed_min;
  int32_t reserved2;
  int64_t steps_min, steps_max;
} pulse_ztask_task_args_t;
int pulse_ztask_reset_task(const pulse_ztask_task_args_t* args, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Rollout glue of the latent-space tasks (AMPAgent.play_steps, phc/learning/amp_agent.py:341-439, over HumanoidReachZ / HumanoidSpeedZ /
 * HumanoidStrikeZ; HumanoidZ.step -> step_z, phc/env/tasks/humanoid_z.py:157-173), written into experience-buffer slices.
 *
 * pulse_latent_post: what pulse_policy_post followed by pulse_vae_reparam(PULSE_Z_RESIDUAL) do, in one launch, one warp per row:
 *   a_z = mu + exp(logstd) * eps (eps injected, or Philox4x32-10 keyed (seed, row, *rng_offset + rng_step) exactly as
 *   pulse_policy_post draws it), neglogp, the de-normalised value (running_mean_std.py:84-87), and z = prior_mu + a_z
 *   (HumanoidZ.compute_z_actions, humanoid_z.py:104-107) as bf16 into the decoder operand's latent columns.  Every output is bit-equal
 *   to the two-launch composition.  pulse_z_task.yaml has clip_actions False and project_to_norm(.., "none") is the identity, so a_z is
 *   neither clamped nor projected.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* mu; int64_t ld_mu;            /* [rows, latent] latent policy head output */
  const float* logstd;                       /* [latent] */
  const float* eps; int64_t ld_eps;          /* [rows, latent] injected standard-normal draws, or NULL -> Philox */
  uint64_t seed; const uint64_t* rng_offset; uint64_t rng_step;
  int32_t latent; int32_t reserved;          /* 1 .. 128 */
  float* actions; int64_t ld_actions;        /* out: a_z */
  float* neglogp; int64_t ld_neglogp;        /* out, element stride */
  const float* value; int64_t ld_value;      /* [rows] normalised critic output */
  const double* value_mean; const double* value_var; float value_eps; int32_t reserved2;   /* RunningMeanStd of the value (NULL = identity) */
  float* values_out; int64_t ld_values;      /* out */
  const float* prior_mu; int64_t ld_prior;   /* [rows, >= latent] frozen prior head; columns [0, latent) = prior mean */
  pulse_bf16_t* z_bf16; int64_t ld_z;        /* out: z into columns [0, latent) of the decoder operand rows */
} pulse_latent_post_args_t;
int pulse_latent_post(const pulse_latent_post_args_t* args, int64_t rows, void* stream);

/* pulse_ztask_pre_physics: the pre-physics work of one latent-task step over num_envs envs in one launch:
 *   pd_out[e, d]   = freeze[d] ? 0 : pd_offset[d] + pd_scale[d] * action[e, d]      (pulse_pd_targets' arithmetic; humanoid.py:1222-1247)
 *   prev_root_pos[e] = root_states[e, 0:3]                                          (speed, strike; humanoid_speed.py:73-76)
 *   _update_task where progress_buf[e] >= change_steps[e]   (reach humanoid_reach.py:127-146, speed humanoid_speed.py:157-175):
 *     PULSE_ZTASK_REACH  tar_pos = (dist_max (2u - 1), dist_max (2v - 1), (height_max - height_min) w + height_min), the arithmetic of
 *                        pulse_reach_update_task
 *     PULSE_ZTASK_SPEED  tar_speed = speed_scale u + speed_min (two roundings, as the tensor expression of the reference)
 *     change_steps = progress + randint(steps_min, steps_max);  PULSE_ZTASK_STRIKE has no _update_task
 *   Only due envs are written.  Draws: injected per ENV (rand: reach [N, 3], speed [N]; steps_in int64 [N]) or the Philox4x32-10 words of
 *     index e + 3 * 2^32   x, y, z task uniforms, w change steps (steps_min + (w (steps_max - steps_min)) >> 32)
 *   on (seed, index, offset + *offset_dev): a fourth index plane beside the three of pulse_reset_ztask / pulse_ztask_reset_task
 *   (e, e + 2^32, e + 2^33), so a step that resets an env and later updates its task draws from different words. */
typedef struct {
  int32_t kind; int32_t dofs;
  const float* action; int64_t ld_action;    /* [N, dofs] decoder output */
  const float* pd_offset; const float* pd_scale; const uint8_t* freeze;   /* [dofs]; freeze may be NULL */
  float* pd_out; int64_t ld_pd;
  const float* root_states; int64_t root_env_stride; float* prev_root_pos;   /* speed, strike: [N, >= 3] view, [N, 3]; NULL for reach */
  const int64_t* progress_buf;
  int64_t* change_steps;                     /* reach, speed: _tar_change_steps / _speed_change_steps */
  float* tar_pos;                            /* reach [N, 3] */
  float* tar_speed;                          /* speed [N] */
  const float* rand;                         /* injected uniforms, or NULL: Philox */
  const int64_t* steps_in;                   /* injected randint results, or NULL: Philox */
  uint64_t seed, offset;
  const uint64_t* offset_dev;
  float dist_max, height_min, height_max, speed_scale, speed_min;
  int32_t reserved;
  int64_t steps_min, steps_max;
} pulse_ztask_pre_physics_args_t;
int pulse_ztask_pre_physics(const pulse_ztask_pre_physics_args_t* args, int64_t num_envs, void* stream);

/* Post-physics step of the rollout (humanoid.py:1315-1346): `progress_buf += 1` inside the kernel (the argument structs' progress_buf is
 * written here), then the per-env code of pulse_reach_step / pulse_ztask_step, then dones[e] = float(reset_buf[e]) (amp_agent.py:380).
 * obs_buf / obs_stride address the next step's experience slice, rew_buf the step's reward row.  Outputs are bit-equal to advancing
 * the counter and calling the plain step. */
int pulse_reach_rollout_step(const pulse_reach_step_args_t* args, float* dones, int64_t num_envs, void* stream);
int pulse_ztask_rollout_step(const pulse_ztask_step_args_t* args, float* dones, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The PULSE-X speed task: HumanoidSpeedZ with robot=smplx_humanoid, env_pulsex_amp.yaml, learning=pulse_z_task.yaml.  The 52-body
 * SMPL-X humanoid (bodies in SMPLH_MUJOCO_NAMES order, humanoid.py:376-377; body 0 the root; 51 joints x 3 = 153 dofs), beside the
 * SMPL entry points above, which it leaves unchanged.  Body sets (contact bodies, termination heights) arrive as arguments; no
 * entry point knows a body name.  The per-env device code is the SMPL step's and reset's, instantiated for 52 bodies: one warp per
 * env, lane l holding bodies l and l + 32.
 * ---------------------------------------------------------------------------------------------- */
#define PULSE_SMPLX_BODIES 52
#define PULSE_SMPLX_DOF 153          /* 51 joints x 3                                               */
#define PULSE_SMPLX_SELF_OBS 778     /* 1 + 51*3 + 52*6 + 52*3 + 52*3, humanoid.py:1675-1731          */
#define PULSE_SMPLX_SPEED_OBS 781    /* + compute_speed_observations (humanoid_speed.py:310-325)      */
#define PULSE_SMPLX_FRAME_REC 676    /* packed per-frame record: pos156 | rot208 | vel156 | angvel156 */
#define PULSE_SMPLX_AUX_REC 364      /* packed per-frame record: lrs208 | dvs153 | pad3             */
/* The AMP observation of the SMPL-X humanoid (build_amp_observations_smpl, humanoid_amp.py:924-969, env_pulsex_amp.yaml): dof_subset
 * drops only L_Toe and R_Toe (humanoid.py:404-421), so 49 of the 51 joints are kept; key bodies R_Ankle, L_Ankle, R_Wrist, L_Wrist
 * = bodies 7, 3, 36, 17.  [h 1 | root rot 6 | root vel 3 | root ang vel 3 | 49 x six(dof) | 147 dof vel | 4 x key pos 3], all in
 * the heading frame of remove_base_rot(root_rot) (has_upright_start False); 465 without the root height (ampRootHeightObs False,
 * the env_pulsex_amp.yaml width, 10 x 465 = 4650 floats per discriminator row). */
#define PULSE_SMPLX_AMP_OBS 466
#define PULSE_SMPLX_AMP_OBS_NO_HEIGHT 465

/* MotionLib tables of the SMPL-X humanoid (MotionLibSMPL loaded with smplx_humanoid.xml, motion_lib_base.py:287-316), packed into
 * the two records above by one kernel.  The handle is its own type: SMPL-X tables never reach an SMPL entry point. */
typedef struct pulse_smplx_motionlib pulse_smplx_motionlib_t;
typedef struct {
  const float* gts;   /* [F,52,3] */
  const float* grs;   /* [F,52,4] */
  const float* lrs;   /* [F,52,4] */
  const float* gvs;   /* [F,52,3] */
  const float* gavs;  /* [F,52,3] */
  const float* dvs;   /* [F,51,3] */
  const float* lengths; const float* dt; const int64_t* num_frames; const int64_t* length_starts;   /* [M] */
  int64_t total_frames, num_motions;
  float* frame_rec;   /* [F, PULSE_SMPLX_FRAME_REC], 16-byte aligned, filled by pulse_smplx_motionlib_create */
  float* aux_rec;     /* [F, PULSE_SMPLX_AUX_REC],   16-byte aligned */
} pulse_smplx_motionlib_desc_t;
int pulse_smplx_motionlib_create(const pulse_smplx_motionlib_desc_t* desc, void* stream, pulse_smplx_motionlib_t** out);
int pulse_smplx_motionlib_destroy(pulse_smplx_motionlib_t* lib);

/* get_motion_state (motion_lib_base.py:434-517) over the SMPL-X tables, the arithmetic of pulse_motion_state.  Any output may be NULL. */
typedef struct {
  const int64_t* motion_ids;   /* [n] */
  const float* motion_times;   /* [n] */
  const float* offset;         /* [n,3] or NULL */
  float* root_pos; float* root_rot; float* root_vel; float* root_ang_vel;   /* [n,3] / [n,4] */
  float* dof_pos; float* dof_vel;                                            /* [n,153] */
  float* rg_pos; float* rb_rot; float* body_vel; float* body_ang_vel;       /* [n,52,3] / [n,52,4] */
} pulse_smplx_motion_query_t;
int pulse_smplx_motion_state(const pulse_smplx_motionlib_t* lib, const pulse_smplx_motion_query_t* q, int64_t n, void* stream);

/* Post-physics step of the SMPL-X speed task: the self observation of compute_humanoid_observations_smpl_max with local root obs,
 * root height and has_upright_start False (the heading of remove_base_rot(root_rot), humanoid.py:1617-1620, :1682-1684), then
 * compute_speed_observations, whose heading is that of the RAW root rotation, compute_speed_reward and compute_humanoid_reset.
 * obs[env] = [self 778 | heading-frame x axis 2 | target speed 1].  env_pulsex_amp.yaml has power_reward and power_usage_reward off;
 * this step has neither term.  reward_raw (optional) receives the speed reward. */
typedef struct {
  int32_t enable_early_termination, reserved;
  const float* body_state; int64_t body_env_stride;        /* [N, >=52, 13] pos quat(xyzw) linvel angvel */
  const float* contact_forces; int64_t contact_env_stride; /* [N, >=52, 3] or NULL */
  const float* termination_heights;                        /* [52] */
  uint64_t contact_body_mask;                              /* bit j: body j may touch the ground (_contact_body_ids) */
  const int64_t* progress_buf; int64_t max_episode_length;
  const float* prev_root_pos; float dt; float reserved2;   /* [N, 3] root position before the physics step */
  const float* tar_speed;                                  /* [N] */
  float* obs_buf; int64_t obs_stride;                      /* [N, >= 781] */
  float* rew_buf; float* reward_raw; int64_t raw_stride;
  int64_t* reset_buf; int64_t* terminate_buf;
} pulse_smplx_speed_step_args_t;
int pulse_smplx_speed_step(const pulse_smplx_speed_step_args_t* args, int64_t num_envs, void* stream);
/* The observation rows of the envs env_list[0 .. *count), as pulse_ztask_obs_list. */
int pulse_smplx_speed_obs_list(const pulse_smplx_speed_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs,
                               void* stream);
/* progress_buf += 1, the step, dones[e] = float(reset_buf[e]), as pulse_ztask_rollout_step. */
int pulse_smplx_speed_rollout_step(const pulse_smplx_speed_step_args_t* args, float* dones, int64_t num_envs, void* stream);

/* Post-physics step of the SMPL-X reach and strike tasks (HumanoidReachZ / HumanoidStrikeZ with robot=smplx_humanoid): the self
 * observation of pulse_smplx_speed_step (the heading of remove_base_rot(root_rot)), then the task observation in the heading of the
 * RAW root rotation, the reward and the reset, as the SMPL steps compute them:
 *   PULSE_ZTASK_REACH   compute_location_observations / compute_reach_reward (humanoid_reach.py:224-250), reward
 *                       exp(-4 ||tar_pos - p[reach_body_id]||^2); compute_humanoid_reset (humanoid.py:1573-1608).  obs 778 + 3.
 *   PULSE_ZTASK_STRIKE  compute_strike_observations / compute_strike_reward (humanoid_strike.py:270-328), the strike variant of
 *                       compute_humanoid_reset (:330-375): also fails when the target is pushed (> 50 N in x or y) while a body in
 *                       neither contact_body_mask nor strike_body_mask presses harder than 50 N, over all 52 bodies.  obs 778 + 15.
 * Body sets are 64-bit masks (SMPL-X body ids go up to 51; bits 52..63 must be clear).  Neither task has a power term. */
#define PULSE_SMPLX_REACH_OBS 781    /* 778 + compute_location_observations 3 */
#define PULSE_SMPLX_STRIKE_OBS 793   /* 778 + compute_strike_observations 15  */
typedef struct {
  int32_t kind, enable_early_termination;                  /* PULSE_ZTASK_REACH or PULSE_ZTASK_STRIKE */
  const float* body_state; int64_t body_env_stride;        /* [N, >=52, 13] pos quat(xyzw) linvel angvel */
  const float* contact_forces; int64_t contact_env_stride; /* [N, >=52, 3] or NULL */
  const float* termination_heights;                        /* [52] */
  uint64_t contact_body_mask;                              /* bit j: body j may touch the ground (_contact_body_ids) */
  uint64_t strike_body_mask;                               /* strike: bit j: body j may hit the target (_strike_body_ids) */
  int32_t reach_body_id; int32_t reserved;                 /* reach: [0, 52) */
  const int64_t* progress_buf; int64_t max_episode_length;
  const float* tar_pos;                                    /* reach: [N, 3] */
  const float* prev_root_pos; float dt; float reserved2;   /* strike: [N, 3] root position before the physics step */
  const float* target_states; int64_t target_env_stride;   /* strike: [N, 13] view of the target actor's root state */
  const float* tar_contact_forces; int64_t tar_contact_env_stride;   /* strike: [N, 3] view */
  float* obs_buf; int64_t obs_stride;                      /* [N, >= 781 (reach) / 793 (strike)] */
  float* rew_buf;                                          /* [N] */
  int64_t* reset_buf; int64_t* terminate_buf;              /* [N] */
} pulse_smplx_target_step_args_t;
int pulse_smplx_target_step(const pulse_smplx_target_step_args_t* args, int64_t num_envs, void* stream);
/* The observation rows of the envs env_list[0 .. *count), as pulse_ztask_obs_list. */
int pulse_smplx_target_obs_list(const pulse_smplx_target_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs,
                                void* stream);
/* progress_buf += 1, the step, dones[e] = float(reset_buf[e]), as pulse_ztask_rollout_step. */
int pulse_smplx_target_rollout_step(const pulse_smplx_target_step_args_t* args, float* dones, int64_t num_envs, void* stream);

/* The reference-state reset of pulse_reset_ztask for the SMPL-X speed task, no host synchronisation: the compaction, then one warp per
 * (reset env, AMP history step k): clip and start-time draws, the 52-body gather, the SMPL ground fix from the per-frame floor table,
 * the FACE_X pose adjustment (HumanoidSpeed._sample_ref_state, humanoid_speed.py:251-270, heading of remove_base_rot(root_rot) when
 * !upright) and the scatter into the root, [N, >= 52, 13] rigid-body and [N, 153] dof views, counters and contact forces.  The argument
 * struct is pulse_reset_ztask's with pose_mode PULSE_ZPOSE_FACE_X; the strike target (target_states) is refused.  With amp_obs_buf
 * [N, num_amp_steps, amp_width] (amp_width PULSE_SMPLX_AMP_OBS or PULSE_SMPLX_AMP_OBS_NO_HEIGHT, num_amp_steps 1..16) the AMP history
 * is back-filled as in pulse_reset_ztask: row 0 from the state just written, rows k >= 1 from the unadjusted motion at t0 - k dt; the
 * state outputs are those of the same call without it.  _reset_task follows through pulse_ztask_reset_task, the PD targets through
 * pulse_ztask_pre_physics (dofs 153). */
int pulse_reset_ztask_smplx(const pulse_smplx_motionlib_t* lib, const pulse_ztask_reset_args_t* args, int64_t num_envs, void* stream);

/* The reference-state reset of pulse_reset_ztask_smplx for the SMPL-X reach and strike tasks: the same launches and checks, with
 * pose_mode PULSE_ZPOSE_ROOT_XY_ZERO (humanoid_reach.py:46-48, humanoid_strike.py:147-150; any other mode is refused).  target_states
 * is NULL for reach and the [N, 13] target view for strike, which receives _reset_target (humanoid_strike.py:124-145) around the new
 * root as in pulse_reset_ztask, with the same draws.  _reset_task of the reach task follows through pulse_ztask_reset_task. */
int pulse_reset_smplx_target(const pulse_smplx_motionlib_t* lib, const pulse_ztask_reset_args_t* args, int64_t num_envs, void* stream);

/* pulse_amp_obs_row for the SMPL-X humanoid: the AMP row [current W | first (steps-1)*W floats of the previous row] of every env from
 * [N, >= 52, 13] body views and [N, 153] dof views, W = amp_width PULSE_SMPLX_AMP_OBS or PULSE_SMPLX_AMP_OBS_NO_HEIGHT (0 is refused),
 * with the heading of remove_base_rot(q0) (remove_base_rot must be 1); fresh envs take their history from fresh_rows, as there. */
int pulse_smplx_amp_obs_row(const pulse_amp_row_args_t* args, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Pedestrian terrain task HumanoidPedestrianTerrain(Z) (phc/env/tasks/humanoid_pedestrian_terrain.py): post_physics_step in one launch,
 * one warp per env, selected by PULSE_STEP_REWARD / RESET / OBS:
 *   reward  _compute_reward :871-896: exp(-2 |tar - actor root|^2_xy) at tar = calc_pos(progress * dt) (fuzzy: errors < 0.0025 -> 0,
 *           :1633-1646); power = -coef * sum |dof_force * dof_vel| always in reward_raw[:, 1], added to rew only with power_reward.
 *   reset   compute_humanoid_reset :1477-1531: |sum of the contact forces of the non-contact bodies| > 50 and progress > 1, or the
 *           rigid-body root farther than fail_dist from tar (xy); no_collision_check clears both; progress >= max_len - 1 resets.
 *   obs     [self 358 | trajectory 2T | heights P]: the self observation with the mean center height around the rigid-body root
 *           subtracted from every body's z (:195-223); trajectory samples at progress * dt + k * traj_sample_timestep in the actor
 *           root's heading frame (:385-440, :1588-1616); heights at the head pose (:296-311, :718-772), clip(ref - h, -3, 3) * 5 with
 *           ref = the mean center height around the actor root (use_center_height) or the actor root's z.
 * Heights: Terrain.world_points_to_map / sample_height_points (:1191-1198, :1261-1267) on the int16 heightfield [rows, cols]
 * (row = x cell), or 0 everywhere for a plane (heightfield NULL).  Trajectories: TrajGenerator.calc_pos (phc/utils/traj_generator.py:
 * 148-165) on traj_verts [N, PULSE_TRAJ_VERTS, 3]; traj_dur = num_verts * the generator's dt (the reference's divisor).
 * env_ids (+ optional device-side env_count) restricts an OBS-only call to the listed envs (_compute_observations(env_ids)).
 * Not covered: group observations, the velocity map, mesh terrain, shape observations.
 * ---------------------------------------------------------------------------------------------- */
#define PULSE_TRAJ_VERTS 101
#define PULSE_TRAJ_DRAWS (4 * (PULSE_TRAJ_VERTS - 1) + 2)
#define PULSE_TERRAIN_OBS 1402      /* 358 + 2 * 10 + 32 * 32 (env_pulse_terrain.yaml) */
typedef struct {
  uint32_t flags;                                            /* PULSE_STEP_REWARD | PULSE_STEP_RESET | PULSE_STEP_OBS */
  int32_t upright;                                           /* _has_upright_start (else remove_base_rot) */
  const float* body_state; int64_t body_env_stride;          /* rigid bodies [N, >=24, 13] */
  const float* root_states; int64_t root_env_stride;         /* actor root state [N, 13] view (_humanoid_root_states) */
  const int64_t* progress_buf; int64_t max_episode_length;
  const float* contact_forces; int64_t contact_env_stride;   /* [N, >=24, 3] */
  uint32_t contact_body_mask;                                /* _contact_body_ids */
  int32_t enable_early_termination, no_collision_check, fuzzy_target, power_reward;
  int32_t num_traj_samples, num_height_points, num_center_points, head_body_id, use_center_height;
  float dt, traj_dur, traj_sample_timestep, fail_dist, power_coefficient;
  const float* traj_verts;                                   /* [N, PULSE_TRAJ_VERTS, 3] */
  const int16_t* heightfield; int64_t hf_rows, hf_cols;      /* NULL = plane */
  float horizontal_scale, vertical_scale;
  const float* height_points;                                /* [num_height_points, 3] sensor offsets (square / fov / square_fov) */
  const float* center_points;                                /* [num_center_points, 3] (the 3 x 3 grid of init_center_height_points) */
  const float* dof_force; int64_t dof_force_stride;          /* [N, 69]: the power term; required with power_reward or reward_raw */
  const float* dof_vel; int64_t dof_env_stride, dof_elem_stride;
  const int64_t* env_ids; const int32_t* env_count;          /* optional, OBS only */
  float* obs_buf; int64_t obs_stride;
  float* rew_buf; float* reward_raw; int64_t raw_stride;     /* reward_raw [N, 2] or NULL */
  int64_t* reset_buf; int64_t* terminate_buf;
} pulse_terrain_step_args_t;
int pulse_terrain_step(const pulse_terrain_step_args_t* args, int64_t num_envs, void* stream);

/* Post-physics step of the terrain task's rollout (humanoid.py:1315-1346): `progress_buf += 1` inside the kernel (the struct's
 * progress_buf is written here; the new value is broadcast to the env's warp, which never reads the counter from memory), then the
 * per-env code of pulse_terrain_step with flags PULSE_STEP_ALL (the only flags accepted; no env_ids), then dones[e] =
 * float(reset_buf[e]) (amp_agent.py:380).  obs_buf / obs_stride address the next step's experience slice, rew_buf the step's reward
 * row.  Argument checks as pulse_terrain_step, plus dones != NULL.  Outputs are bit-equal to advancing the counter and calling
 * pulse_terrain_step(PULSE_STEP_ALL). */
int pulse_terrain_rollout_step(const pulse_terrain_step_args_t* args, float* dones, int64_t num_envs, void* stream);

/* TrajGenerator.reset (phc/utils/traj_generator.py:57-112) for num_ids envs, one thread each: random turns (sharp turns with
 * probability sharp_turn_prob), the clipped speed recurrence, waypoints from init_pos's xy (row i belongs to env_ids[i]).  rand
 * [num_ids, PULSE_TRAJ_DRAWS] injects the uniform draws (layout in terrain.cu); NULL draws them with Philox4x32-10 keyed by
 * (seed, env, offset + *offset_dev + k), k < PULSE_TRAJ_VERTS -- a different stream from torch's generator, the same distribution.
 * dtheta_scale = dtheta_max * dt, dspeed_scale = accel_max * dt, seg_dt = dt, with dt = episode_dur / (num_verts - 1). */
typedef struct {
  const int64_t* env_ids; int64_t num_ids;
  const float* init_pos; int64_t init_stride;
  const float* rand;
  uint64_t seed, offset; const uint64_t* offset_dev;
  float dtheta_scale, dspeed_scale, seg_dt, speed_min, speed_max, sharp_turn_prob;
  float* verts;                                              /* [N, PULSE_TRAJ_VERTS, 3] */
} pulse_traj_reset_args_t;
int pulse_traj_reset(const pulse_traj_reset_args_t* args, void* stream);

/* get_center_heights (PULSE_HEIGHTS_CENTER: points rotated by the yaw of the root, quat_apply_yaw :1571-1576) or get_heights
 * (PULSE_HEIGHTS_GRID: by calc_heading_quat) for num_rows root states [pos 3 | quat 4], heights [num_rows, num_points]. */
#define PULSE_HEIGHTS_CENTER 1
#define PULSE_HEIGHTS_GRID 2
typedef struct {
  int32_t mode, upright;
  const float* root_states; int64_t root_stride; int64_t num_rows;
  const float* points; int64_t num_points;
  const int16_t* heightfield; int64_t hf_rows, hf_cols;
  float horizontal_scale, vertical_scale;
  float* heights; int64_t heights_stride;
} pulse_terrain_heights_args_t;
int pulse_terrain_heights(const pulse_terrain_heights_args_t* args, void* stream);

/* pulse_traj_reset_list: TrajGenerator.reset (phc/utils/traj_generator.py:57-112) over the env list and device-side count of a reset
 * (pulse_reset_terrain's env_list / count), one thread per listed env, starting at root_states[e, 0:2] (_reset_task,
 * humanoid_pedestrian_terrain.py:480-485, reads _humanoid_root_states after the reset).  rand [N, PULSE_TRAJ_DRAWS] injects the draws
 * per ENV (layout of pulse_traj_reset); NULL takes them from Philox4x32-10 on (seed, e + 4 * 2^32, PULSE_TRAJ_VERTS * (offset +
 * *offset_dev) + k): two resets of one env at different offsets never share a block.  Parameters as pulse_traj_reset. */
typedef struct {
  const int64_t* env_list; const int32_t* count;
  const float* root_states; int64_t root_env_stride;         /* [N, >= 2] view: the start xy */
  const float* rand;                                         /* [N, PULSE_TRAJ_DRAWS] or NULL */
  uint64_t seed, offset; const uint64_t* offset_dev;
  float dtheta_scale, dspeed_scale, seg_dt, speed_min, speed_max, sharp_turn_prob;
  float* verts;                                              /* [N, PULSE_TRAJ_VERTS, 3] */
} pulse_traj_list_args_t;
int pulse_traj_reset_list(const pulse_traj_list_args_t* args, int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Reference-state reset of the pedestrian terrain task, free of host synchronisation: HumanoidPedestrianTerrain._reset_ref_state_init
 * (humanoid_pedestrian_terrain.py:527-589) with _sample_ref_state (:488-525), _set_env_state, _reset_env_tensors and _init_amp_obs,
 * for humanoid_type "smpl".  The launches and the per-warp work of pulse_reset_ztask (args as there, pose_mode AS_IS, state_init
 * RANDOM: the terrain task's _sample_ref_state always calls _sample_time, for StateInit Start too; no strike target), with the
 * spawn in place of the pose adjustment:
 *   - location: Terrain.sample_valid_locations (:1175-1189), new_xy = (coord_x[l], coord_y[l]) with l injected per env
 *     (loc_ids_in, the np.random.randint draw) or (word z * num_locations) >> 32; l is written to loc_ids_out when given;
 *   - diff = new_xy - root_xy; root_xy = new_xy; root_z += mean of get_center_heights at the new root (:690-716: the center points
 *     rotated by the yaw of the root, or of remove_base_rot(root) when !upright);
 *   - rigid-body xy += diff.  The rigid bodies' z is NOT lifted (the reference adds the lift to key_pos only, twice, and never
 *     reads key_pos again), so AMP row 0, built from the rigid bodies, carries the unlifted root height.
 * The walkable table is Terrain.__init__'s (:1160-1171): the cells with walkable_field == 0 inside the border, scaled by
 * horizontal_scale.  A plane (heightfield NULL) has no table: the reference cannot spawn on it and neither can this entry point.
 * The observation of the reset envs follows (pulse_terrain_step, PULSE_STEP_OBS over env_list / count), then
 * pulse_traj_reset_list, as in the reference (humanoid.py:574-587, humanoid_amp_task.py:73-76).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const int16_t* heightfield; int64_t hf_rows, hf_cols;      /* required (no plane) */
  float horizontal_scale, vertical_scale;
  const float* center_points; int64_t num_center_points;     /* [num_center_points, 3], 1 ..= 32 */
  const float* coord_x; const float* coord_y;                /* [num_locations] walkable table (coord_{x,y}_scale) */
  int64_t num_locations;                                     /* 1 .. 2^32 - 1 */
  const int64_t* loc_ids_in;                                 /* [N] injected location index per env (clamped to the table), or NULL */
  int64_t* loc_ids_out;                                      /* [N] out: the location index of each reset env; may be NULL */
} pulse_terrain_spawn_args_t;
int pulse_reset_terrain(const pulse_motionlib_t* lib, const pulse_ztask_reset_args_t* args, const pulse_terrain_spawn_args_t* spawn,
                        int64_t num_envs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * AMP demo and replay rings on the device (learning/replay_buffer.py ReplayBuffer; AMPAgent._init_amp_demo_buf, _update_amp_demos,
 * _store_replay_amp_obs and the buffer samples of train_epoch, phc/learning/amp_agent.py:476-484, :988-1000, :1043-1057), with every
 * counter on the device so that no call reads anything back to the host.  A ring is `capacity` rows of `row_floats` floats and the
 * int64 counters ctr[PULSE_RING_CTRS]:
 *   head, total_count, sample_head   the ReplayBuffer's _head, _total_count, _sample_head;
 *   perm_key                         the number of _reset_sample_idx calls: the sampling permutation _sample_idx is the keyed Feistel
 *                                    bijection of [0, capacity) with round keys Philox(seed, 9 * 2^32, perm_key), cycle-walked;
 *   draws                            the number of fetches / stores (the counter of their Philox draws);
 *   last_count                       the rows the last replay store kept (scratch of pulse_amp_replay_store).
 * The Feistel network: the smallest even bit width 2h >= max(2, ceil(log2 m)) over the domain [0, m); four rounds
 * (L, R) <- (R, L ^ (F(R, k_r) & (2^h - 1))) with F(x, k) = fmix32(x * 0x9E3779B1 ^ k) (MurmurHash3's finaliser), repeated until the
 * value falls inside [0, m).
 * pulse_amp_demo_fetch   fetch_amp_obs_demo + build_amp_obs_demo (phc/env/tasks/humanoid_amp.py:215-284) of num_samples rows straight
 *                        into the ring, then store()'s head / total_count update: per row a clip (inverse CDF of sampling_cdf), t0 by
 *                        sample_time_interval (the SMPL _sample_time, :376-380), the motion at t0 - k dt for k < num_steps without the
 *                        ground fix, build_amp_observations_smpl in amp_width 196 / 195 and the upright setting.  24-body SMPL.
 * pulse_smplx_amp_demo_fetch  the same over the SMPL-X tables: amp_width PULSE_SMPLX_AMP_OBS / PULSE_SMPLX_AMP_OBS_NO_HEIGHT, upright 0;
 *                        the same Philox planes, so clips and start times are pulse_amp_demo_fetch's word for word.
 * pulse_amp_replay_store _store_replay_amp_obs: once total_count > capacity a Bernoulli(keep_prob) keep mask, the ordered compaction of
 *                        the kept rows, a random subset of capacity rows (Feistel permutation of the kept count, subset keys) when more
 *                        survive, then the ring write with wrap and the counter update.
 * pulse_amp_ring_sample  sample(n): positions sample_head + j mod capacity through the permutation, `% head` while total_count <
 *                        capacity, `fallback` row j (the agent's own rows) while the ring is empty; only the sample rows j with
 *                        j mod block < take are gathered (the first `take` rows of every `block`-row minibatch), but sample_head moves by
 *                        the whole n (and to 0 with a new perm_key once it reaches capacity), as the reference's sample(n) does.
 * ---------------------------------------------------------------------------------------------- */
#define PULSE_PLANE_DEMO_CLIP 5
#define PULSE_PLANE_DEMO_TIME 6
#define PULSE_PLANE_REPLAY_KEEP 7
#define PULSE_PLANE_REPLAY_SUBSET 8
#define PULSE_PLANE_RING_PERM 9
#define PULSE_RING_HEAD 0
#define PULSE_RING_TOTAL 1
#define PULSE_RING_SAMPLE_HEAD 2
#define PULSE_RING_PERM_KEY 3
#define PULSE_RING_DRAWS 4
#define PULSE_RING_LAST_COUNT 5
#define PULSE_RING_CTRS 8

typedef struct {
  float* rows;                   /* [capacity, row_floats] */
  int64_t capacity;              /* buffer_size, 1 .. 2^31 - 1 */
  int64_t* ctr;                  /* [PULSE_RING_CTRS] device counters, zero for a new ring */
  uint64_t seed;                 /* Philox key of the ring's draws */
  int32_t row_floats;            /* num_steps * width */
  int32_t reserved;
} pulse_amp_ring_t;

typedef struct {
  pulse_amp_ring_t ring;
  const float* sampling_cdf;     /* [num_motions] inclusive fp32 prefix sum of _sampling_batch_prob */
  int64_t num_samples;           /* rows fetched, <= capacity */
  int32_t num_steps;             /* numAMPObsSteps, 1 .. 16 */
  int32_t amp_width;             /* 196 or 195 (SMPL-X: 466 or 465) */
  int32_t upright;               /* _has_upright_start */
  float dt;                      /* control dt */
  int64_t* motion_ids_out;       /* [num_samples] optional: the drawn clips */
  float* times_out;              /* [num_samples] optional: the drawn t0 */
} pulse_amp_demo_args_t;
int pulse_amp_demo_fetch(const pulse_motionlib_t* lib, const pulse_amp_demo_args_t* args, void* stream);
int pulse_smplx_amp_demo_fetch(const pulse_smplx_motionlib_t* lib, const pulse_amp_demo_args_t* args, void* stream);

typedef struct {
  pulse_amp_ring_t ring;
  const float* src;              /* [num_rows, row_floats] contiguous rows of the horizon (batch_dict['amp_obs']) */
  int64_t num_rows;              /* < 2^31 */
  float keep_prob;               /* amp_replay_keep_prob */
  int32_t reserved;
  int32_t* kept;                 /* [num_rows] scratch: the kept row ids, ascending */
  int64_t* src_rows_out;         /* [min(num_rows, capacity)] optional: the source row of the i-th stored row, -1 past the stored count */
} pulse_amp_store_args_t;
int pulse_amp_replay_store(const pulse_amp_store_args_t* args, void* stream);

typedef struct {
  pulse_amp_ring_t ring;
  int64_t n;                     /* rows of the reference's sample(n); a multiple of block */
  int64_t block, take;           /* gather sample rows j with j mod block < take, 1 <= take <= block */
  const float* fallback;         /* [n, row_floats] rows used while total_count == 0 (sample_head then stays), or NULL: zeros */
  float* out;                    /* [n / block * take, row_floats] */
  int64_t* ring_rows_out;        /* [n / block * take] optional: the ring row of each gathered row, -1 for a fallback row */
} pulse_amp_sample_args_t;
int pulse_amp_ring_sample(const pulse_amp_sample_args_t* args, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Task observation for every observation version / tracked-body subset / number of future samples (SURVEY 8f-4): replaces the
 * dispatch of HumanoidIm._compute_task_obs (phc/env/tasks/humanoid_im.py:757-833) over compute_imitation_observations (:1222-1258,
 * obs_v 1), _v2 (:1261-1301), _v3 (:1304-1326), _v6 (:1328-1378, obs_v 4 / 6), _v7 (:1381-1413), _v8 (:1415-1479, time_steps 1) and
 * _v9 (:1482-1540) on the `_track_bodies_id` rows.  The reference states are the outputs of pulse_motion_state for the N * time_steps
 * sample times in repeat_interleave order (row env * time_steps + t; fut_tracks, humanoid_im.py:723-729), full 24-body arrays.
 * Not covered: zero_out_far / occlusion rewrites (:763-784), the one-hot suffix of obs_v 5, the multi-sample branches of v2 / v8.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* body_state; int64_t body_env_stride;   /* [N, B>=24, 13] rigid-body state view */
  const int32_t* track_ids;                            /* [num_track] device array of body indices < 24; [0] = 0 for versions 2 and 9 */
  int32_t num_track, time_steps, version, upright;     /* upright = _has_upright_start */
  const float* ref_pos; const float* ref_rot; const float* ref_vel; const float* ref_ang_vel;   /* [N * time_steps, 24, 3 | 4] */
  const float* dof_pos; int64_t dof_env_stride, dof_elem_stride;   /* version 2: simulator dof positions (view strides) */
  const float* ref_dof_pos;                            /* version 2: [N, 69] */
  float* obs; int64_t obs_stride;                      /* [N, >= pulse_task_obs_size] */
  int64_t num_envs;
} pulse_task_obs_args_t;
int pulse_task_obs_size(int32_t version, int32_t num_track, int32_t time_steps);   /* floats per env, -1 for an unknown version */
int pulse_im_task_obs(const pulse_task_obs_args_t* args, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Evaluation metrics on the device (SURVEY 8f-2).  One call per evaluation step replaces the per-step bookkeeping of
 * IMAmpAgent._post_step_eval (phc/learning/im_amp.py:244-363: termination state :249-251, the curr_max stopping rule :252-268, :275,
 * the per-sequence `[:(num_steps - 1)]` frame slices :283-287) and the per-frame metrics compute_metrics_lite derives from the
 * frames the reference copies to the host every step (humanoid_im.py:664-673; smpl_sim [3P]): global / root-relative /
 * Procrustes-aligned MPJPE, velocity and acceleration errors -- accumulated into per-env fp64 sums (metres) and frame counts.
 *   ctrl int32[8], zeroed at the start of a chunk: [0] steps taken, [1] chunk finished (later calls are no-ops), [2..4] scratch.
 *   terminate_state int32[N], hist float[N,2,24,3], sums double[N,5] (mpjpe_g, mpjpe_l, mpjpe_pa, vel, accel), counts int32[N,3]
 *   (frames behind sums 0-2, 3, 4): zeroed at the start of a chunk.  bound: envs [0, bound) hold distinct clips (wrapped last chunk,
 *   im_amp.py:254-262), otherwise num_envs.  max_steps_all = max(num_steps).  mpjpe_out float[N] (optional): extras['mpjpe'].
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const float* body_pos; int64_t pos_env_stride, pos_body_stride;     /* body j of env e at body_pos + e*env_stride + j*body_stride */
  const float* body_pos_gt; int64_t gt_env_stride, gt_body_stride;    /* motion_res['rg_pos'] */
  const int64_t* terminate;    /* [N] terminate_buf */
  const int32_t* num_steps;    /* [N] get_motion_num_steps() (motion_lib_base.py:428-432) */
  int32_t num_envs, bound, max_steps_all, reserved;
  int32_t* ctrl; int32_t* terminate_state; float* hist; double* sums; int32_t* counts; float* mpjpe_out;
} pulse_eval_args_t;
int pulse_eval_step(const pulse_eval_args_t* args, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MotionLib loader on the device (SURVEY 8f-1; parity green against the reference's tables, not yet timed).  Per clip: optional heading rotation, local rotations, forward kinematics, gaussian-filtered linear /
 * angular velocities and dof velocities (motion_lib_smpl.py:101-174, poselib skeleton3d.py:389-462, :1100-1118,
 * motion_lib_base.py:47-70) from the on-disk clip arrays concatenated over clips; fills the six fp32 tables
 * pulse_motionlib_create packs.  All pointers are device pointers.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const double* pose_quat_global;  /* [F, 24, 4] xyzw, as stored by convert_amass_isaac.py */
  const double* root_trans;        /* [F, 3] root_trans_offset */
  const int32_t* frame_clip;       /* [F] clip index of every frame */
  const int64_t* clip_start;       /* [M + 1] first frame of every clip, clip_start[M] = F */
  const float* fps;                /* [M] */
  const double* headings;          /* [M] heading angle drawn per clip (motion_lib_smpl.py:134-135), or NULL (im_eval / test) */
  const int32_t* parents;          /* [24] skeleton parent indices (-1 = root) */
  const float* local_translation;  /* [24, 3] skeleton offsets */
  int64_t total_frames, num_clips;
  float* gts; float* grs; float* lrs; float* gvs; float* gavs; float* dvs;   /* outputs, shapes as in pulse_motionlib_desc_t */
  float* tmp_vel; float* tmp_ang;  /* workspaces [F, 24, 3] */
} pulse_loader_args_t;
int pulse_motionlib_load_clips(const pulse_loader_args_t* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PULSE_B200_H_ */
