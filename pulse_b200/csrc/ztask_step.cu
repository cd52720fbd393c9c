// Post-physics step of the downstream latent-space tasks HumanoidReach (SURVEY K21), HumanoidSpeedZ and HumanoidStrikeZ (SURVEY 8f-4):
// one warp per env, lane = body -- self observation (humanoid.py:1675-1731), task observation, reward and reset in one launch.
//   reach   compute_location_observations / compute_reach_reward  phc/env/tasks/humanoid_reach.py:224-250, target resampling
//           (_update_task :126-147) in reach_update_task_kernel, reset = compute_humanoid_reset  humanoid.py:1573-1608
//   speed   compute_speed_observations / compute_speed_reward   phc/env/tasks/humanoid_speed.py:310-343, power term :215-222,
//           reset = compute_humanoid_reset
//   strike  compute_strike_observations / compute_strike_reward  phc/env/tasks/humanoid_strike.py:270-328,
//           reset = the strike variant of compute_humanoid_reset  :330-375
//   smplx speed  the speed step above for the 52-body SMPL-X humanoid (env_pulsex_amp.yaml): the same per-env code instantiated for
//           SmplxLayout, the self observation in the heading of remove_base_rot(root) (has_upright_start False)
//   smplx reach / strike  the reach and strike steps above for the same humanoid (pulse_smplx_target_step): the per-env code
//           instantiated for SmplxTargetLayout, the reach body broadcast from its slot (body id / 32) and lane (body id % 32)
// The per-env device code is ztask_env.cuh's, shared with the rollout step kernels of ztask_rollout.cu.
#include "ztask_env.cuh"

namespace pulse {
namespace {

__global__ void __launch_bounds__(256) reach_update_task_kernel(const long long* __restrict__ progress, long long* __restrict__ change,
                                                                float* __restrict__ tar, const float* __restrict__ u,
                                                                const long long* __restrict__ steps, float dist_max, float h_min, float h_max,
                                                                long long n) {
  for (long long e = blockIdx.x * 256ll + threadIdx.x; e < n; e += 256ll * gridDim.x) {
    if (progress[e] >= change[e]) {
      tar[3 * e + 0] = dist_max * (2.0f * u[3 * e + 0] - 1.0f);
      tar[3 * e + 1] = dist_max * (2.0f * u[3 * e + 1] - 1.0f);
      tar[3 * e + 2] = (h_max - h_min) * u[3 * e + 2] + h_min;
      change[e] = progress[e] + steps[e];
    }
  }
}

__global__ void __launch_bounds__(256) reach_step_kernel(const pulse_reach_step_args_t a, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long e = blockIdx.x * 8ll + warp; e < n; e += 8ll * gridDim.x) reach_env<false>(a, e, lane);
}

__global__ void __launch_bounds__(256) reach_obs_list_kernel(const pulse_reach_step_args_t a, const long long* __restrict__ env_list,
                                                             const int* __restrict__ count) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = *count;
  for (long long i = blockIdx.x * 8ll + warp; i < n; i += 8ll * gridDim.x) reach_env<true>(a, env_list[i], lane);
}

template <class L>
__global__ void __launch_bounds__(256) ztask_step_kernel(const typename L::StepArgs a, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long e = blockIdx.x * 8ll + warp; e < n; e += 8ll * gridDim.x) ztask_env<L, false>(a, e, lane);
}

template <class L>
__global__ void __launch_bounds__(256) ztask_obs_list_kernel(const typename L::StepArgs a, const long long* __restrict__ env_list,
                                                             const int* __restrict__ count) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = *count;
  for (long long i = blockIdx.x * 8ll + warp; i < n; i += 8ll * gridDim.x) ztask_env<L, true>(a, env_list[i], lane);
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_ztask_step(const pulse_ztask_step_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_ztask_step: null args");
  const pulse_ztask_step_args_t& a = *args;
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_SPEED || a.kind == PULSE_ZTASK_STRIKE, "pulse_ztask_step: unknown task kind %d", a.kind);
  PULSE_REQUIRE(num_envs > 0, "pulse_ztask_step: num_envs must be positive");
  PULSE_REQUIRE(a.body_state && a.progress_buf && a.prev_root_pos && a.obs_buf && a.rew_buf && a.reset_buf && a.terminate_buf,
                "pulse_ztask_step: null buffer");
  PULSE_REQUIRE(a.dt > 0.0f, "pulse_ztask_step: dt must be positive");
  PULSE_REQUIRE(a.body_env_stride >= 24 * 13, "pulse_ztask_step: body_env_stride %lld < 312", (long long)a.body_env_stride);
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "pulse_ztask_step: termination_heights required");
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= 24 * 3, "pulse_ztask_step: bad contact stride");
  if (a.kind == PULSE_ZTASK_SPEED) {
    PULSE_REQUIRE(a.tar_speed != nullptr, "pulse_ztask_step: speed task needs tar_speed");
    PULSE_REQUIRE(a.obs_stride >= PULSE_SPEED_OBS, "pulse_ztask_step: obs_stride %lld < %d", (long long)a.obs_stride, PULSE_SPEED_OBS);
    PULSE_REQUIRE(a.dof_force == nullptr || (a.dof_vel != nullptr && a.dof_elem_stride >= 1), "pulse_ztask_step: power term needs dof_vel");
    PULSE_REQUIRE(a.reward_raw == nullptr || a.raw_stride >= (a.dof_force ? 2 : 1), "pulse_ztask_step: raw_stride too small");
  } else {
    PULSE_REQUIRE(a.target_states && a.tar_contact_forces, "pulse_ztask_step: strike task needs target_states and tar_contact_forces");
    PULSE_REQUIRE(a.obs_stride >= PULSE_STRIKE_OBS, "pulse_ztask_step: obs_stride %lld < %d", (long long)a.obs_stride, PULSE_STRIKE_OBS);
  }
  ztask_step_kernel<SmplLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("ztask_step_kernel");
  return PULSE_OK;
}

extern "C" int pulse_reach_update_task(const int64_t* progress, int64_t* tar_change_steps, float* tar_pos, const float* rand01,
                                       const int64_t* steps, float dist_max, float h_min, float h_max, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(progress && tar_change_steps && tar_pos && rand01 && steps, "pulse_reach_update_task: null buffer");
  PULSE_REQUIRE(num_envs > 0, "pulse_reach_update_task: num_envs <= 0");
  reach_update_task_kernel<<<grid_for(num_envs, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(progress), reinterpret_cast<long long*>(tar_change_steps), tar_pos, rand01,
      reinterpret_cast<const long long*>(steps), dist_max, h_min, h_max, num_envs);
  PULSE_LAUNCH_OK("reach_update_task_kernel");
  return PULSE_OK;
}

extern "C" int pulse_reach_step(const pulse_reach_step_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args, "pulse_reach_step: null args");
  const pulse_reach_step_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.tar_pos && a.progress_buf && a.obs_buf && a.rew_buf && a.reset_buf && a.terminate_buf,
                "pulse_reach_step: null buffer");
  PULSE_REQUIRE(num_envs > 0 && a.body_env_stride >= 24 * 13 && a.obs_stride >= PULSE_REACH_OBS, "pulse_reach_step: bad strides");
  PULSE_REQUIRE(a.reach_body_id >= 0 && a.reach_body_id < 24, "pulse_reach_step: reach_body_id out of range");
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "pulse_reach_step: termination_heights required");
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= 24 * 3, "pulse_reach_step: bad contact stride");
  reach_step_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, num_envs);
  PULSE_LAUNCH_OK("reach_step_kernel");
  return PULSE_OK;
}

// The observation of the envs in env_list[0 .. *count): the rows pulse_reach_step / pulse_ztask_step write for them, nothing else.
extern "C" int pulse_reach_obs_list(const pulse_reach_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs,
                                    void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args && env_list && count, "pulse_reach_obs_list: null args / env_list / count");
  const pulse_reach_step_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.tar_pos && a.obs_buf, "pulse_reach_obs_list: null buffer");
  PULSE_REQUIRE(num_envs >= 0 && a.body_env_stride >= 24 * 13 && a.obs_stride >= PULSE_REACH_OBS, "pulse_reach_obs_list: bad strides");
  if (num_envs == 0) return PULSE_OK;
  reach_obs_list_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, reinterpret_cast<const long long*>(env_list), count);
  PULSE_LAUNCH_OK("reach_obs_list_kernel");
  return PULSE_OK;
}

extern "C" int pulse_ztask_obs_list(const pulse_ztask_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs,
                                    void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args && env_list && count, "pulse_ztask_obs_list: null args / env_list / count");
  const pulse_ztask_step_args_t& a = *args;
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_SPEED || a.kind == PULSE_ZTASK_STRIKE, "pulse_ztask_obs_list: unknown task kind %d", a.kind);
  PULSE_REQUIRE(num_envs >= 0 && a.body_state && a.obs_buf && a.body_env_stride >= 24 * 13, "pulse_ztask_obs_list: null buffer or bad stride");
  PULSE_REQUIRE(a.kind != PULSE_ZTASK_SPEED || (a.tar_speed && a.obs_stride >= PULSE_SPEED_OBS), "pulse_ztask_obs_list: speed needs tar_speed, obs_stride >= 361");
  PULSE_REQUIRE(a.kind != PULSE_ZTASK_STRIKE || (a.target_states && a.target_env_stride >= 13 && a.obs_stride >= PULSE_STRIKE_OBS),
                "pulse_ztask_obs_list: strike needs target_states, obs_stride >= 373");
  if (num_envs == 0) return PULSE_OK;
  ztask_obs_list_kernel<SmplLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, reinterpret_cast<const long long*>(env_list), count);
  PULSE_LAUNCH_OK("ztask_obs_list_kernel");
  return PULSE_OK;
}

namespace pulse {
// The checks of the SMPL-X speed step's arguments shared by its three entry points (`who` prefixes the messages).
int check_smplx_speed_args(const pulse_smplx_speed_step_args_t* args, bool step, const char* who) {
  PULSE_REQUIRE(args != nullptr, "%s: null args", who);
  const pulse_smplx_speed_step_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.obs_buf && a.tar_speed, "%s: null body_state / obs_buf / tar_speed", who);
  PULSE_REQUIRE(a.body_env_stride >= PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W, "%s: body_env_stride %lld < %d", who,
                (long long)a.body_env_stride, PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W);
  PULSE_REQUIRE(a.obs_stride >= PULSE_SMPLX_SPEED_OBS, "%s: obs_stride %lld < %d", who, (long long)a.obs_stride, PULSE_SMPLX_SPEED_OBS);
  if (!step) return PULSE_OK;
  PULSE_REQUIRE(a.progress_buf && a.prev_root_pos && a.rew_buf && a.reset_buf && a.terminate_buf, "%s: null buffer", who);
  PULSE_REQUIRE(a.dt > 0.0f, "%s: dt must be positive", who);
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "%s: termination_heights required", who);
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= PULSE_SMPLX_BODIES * 3, "%s: contact_env_stride %lld < %d", who,
                (long long)a.contact_env_stride, PULSE_SMPLX_BODIES * 3);
  PULSE_REQUIRE(a.reward_raw == nullptr || a.raw_stride >= 1, "%s: raw_stride too small", who);
  return PULSE_OK;
}
}  // namespace pulse

extern "C" int pulse_smplx_speed_step(const pulse_smplx_speed_step_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  const int st = check_smplx_speed_args(args, true, "pulse_smplx_speed_step");
  if (st != PULSE_OK) return st;
  PULSE_REQUIRE(num_envs > 0, "pulse_smplx_speed_step: num_envs must be positive");
  ztask_step_kernel<SmplxLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, (long long)num_envs);
  PULSE_LAUNCH_OK("ztask_step_kernel<SmplxLayout>");
  return PULSE_OK;
}

extern "C" int pulse_smplx_speed_obs_list(const pulse_smplx_speed_step_args_t* args, const int64_t* env_list, const int32_t* count,
                                          int64_t num_envs, void* stream) {
  using namespace pulse;
  const int st = check_smplx_speed_args(args, false, "pulse_smplx_speed_obs_list");
  if (st != PULSE_OK) return st;
  PULSE_REQUIRE(env_list && count && num_envs >= 0, "pulse_smplx_speed_obs_list: null env_list / count or negative num_envs");
  if (num_envs == 0) return PULSE_OK;
  ztask_obs_list_kernel<SmplxLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      *args, reinterpret_cast<const long long*>(env_list), count);
  PULSE_LAUNCH_OK("ztask_obs_list_kernel<SmplxLayout>");
  return PULSE_OK;
}

namespace pulse {
// The checks of the SMPL-X reach / strike step's arguments shared by its three entry points (`who` prefixes the messages).
int check_smplx_target_args(const pulse_smplx_target_step_args_t* args, bool step, const char* who) {
  PULSE_REQUIRE(args != nullptr, "%s: null args", who);
  const pulse_smplx_target_step_args_t& a = *args;
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_REACH || a.kind == PULSE_ZTASK_STRIKE, "%s: task kind %d, this step serves PULSE_ZTASK_REACH and "
                "PULSE_ZTASK_STRIKE", who, a.kind);
  const bool reach = a.kind == PULSE_ZTASK_REACH;
  PULSE_REQUIRE(a.body_state && a.obs_buf, "%s: null body_state / obs_buf", who);
  PULSE_REQUIRE(a.body_env_stride >= PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W, "%s: body_env_stride %lld < %d", who,
                (long long)a.body_env_stride, PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W);
  const int width = reach ? PULSE_SMPLX_REACH_OBS : PULSE_SMPLX_STRIKE_OBS;
  PULSE_REQUIRE(a.obs_stride >= width, "%s: obs_stride %lld < %d", who, (long long)a.obs_stride, width);
  PULSE_REQUIRE(!reach || a.tar_pos != nullptr, "%s: the reach task needs tar_pos", who);
  PULSE_REQUIRE(reach || (a.target_states != nullptr && a.target_env_stride >= PULSE_BODY_STATE_W), "%s: the strike task needs "
                "target_states with target_env_stride >= 13", who);
  if (!step) return PULSE_OK;
  PULSE_REQUIRE(a.progress_buf && a.rew_buf && a.reset_buf && a.terminate_buf, "%s: null buffer", who);
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "%s: termination_heights required", who);
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= PULSE_SMPLX_BODIES * 3, "%s: contact_env_stride %lld < %d", who,
                (long long)a.contact_env_stride, PULSE_SMPLX_BODIES * 3);
  PULSE_REQUIRE(((a.contact_body_mask | a.strike_body_mask) >> PULSE_SMPLX_BODIES) == 0, "%s: contact_body_mask / strike_body_mask "
                "set bits at or above %d", who, PULSE_SMPLX_BODIES);
  if (reach) {
    PULSE_REQUIRE(a.reach_body_id >= 0 && a.reach_body_id < PULSE_SMPLX_BODIES, "%s: reach_body_id %d outside [0, %d)", who, a.reach_body_id,
                  PULSE_SMPLX_BODIES);
  } else {
    PULSE_REQUIRE(a.tar_contact_forces != nullptr, "%s: the strike task needs tar_contact_forces", who);
    PULSE_REQUIRE(a.prev_root_pos != nullptr, "%s: the strike task needs prev_root_pos", who);
    PULSE_REQUIRE(a.dt > 0.0f, "%s: dt must be positive", who);
  }
  return PULSE_OK;
}
}  // namespace pulse

extern "C" int pulse_smplx_target_step(const pulse_smplx_target_step_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  const int st = check_smplx_target_args(args, true, "pulse_smplx_target_step");
  if (st != PULSE_OK) return st;
  PULSE_REQUIRE(num_envs > 0, "pulse_smplx_target_step: num_envs must be positive");
  ztask_step_kernel<SmplxTargetLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, (long long)num_envs);
  PULSE_LAUNCH_OK("ztask_step_kernel<SmplxTargetLayout>");
  return PULSE_OK;
}

extern "C" int pulse_smplx_target_obs_list(const pulse_smplx_target_step_args_t* args, const int64_t* env_list, const int32_t* count,
                                           int64_t num_envs, void* stream) {
  using namespace pulse;
  const int st = check_smplx_target_args(args, false, "pulse_smplx_target_obs_list");
  if (st != PULSE_OK) return st;
  PULSE_REQUIRE(env_list && count && num_envs >= 0, "pulse_smplx_target_obs_list: null env_list / count or negative num_envs");
  if (num_envs == 0) return PULSE_OK;
  ztask_obs_list_kernel<SmplxTargetLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      *args, reinterpret_cast<const long long*>(env_list), count);
  PULSE_LAUNCH_OK("ztask_obs_list_kernel<SmplxTargetLayout>");
  return PULSE_OK;
}
