// Post-physics step of the downstream latent-space tasks HumanoidReach (SURVEY K21), HumanoidSpeedZ and HumanoidStrikeZ (SURVEY 8f-4):
// one warp per env, lane = body -- self observation (humanoid.py:1675-1731), task observation, reward and reset in one launch.
//   reach   compute_location_observations / compute_reach_reward  phc/env/tasks/humanoid_reach.py:224-250, target resampling
//           (_update_task :126-147) in reach_update_task_kernel, reset = compute_humanoid_reset  humanoid.py:1573-1608
//   speed   compute_speed_observations / compute_speed_reward   phc/env/tasks/humanoid_speed.py:310-343, power term :215-222,
//           reset = compute_humanoid_reset
//   strike  compute_strike_observations / compute_strike_reward  phc/env/tasks/humanoid_strike.py:270-328,
//           reset = the strike variant of compute_humanoid_reset  :330-375
// One kernel template, ztask_kernel<L, mode>, runs ztask_env.cuh's per-env code for every body layout and argument struct
// (humanoid_obs.cuh): SmplReachLayout (pulse_reach_*), SmplLayout (pulse_ztask_*: speed and strike), SmplxLayout (pulse_smplx_speed_*:
// the 52-body SMPL-X humanoid of env_pulsex_amp.yaml, self observation in the heading of remove_base_rot(root)) and SmplxTargetLayout
// (pulse_smplx_target_*: SMPL-X reach and strike, the reach body broadcast from its slot and lane).  Each layout has three entry
// points, one per mode: the step, the observation of an env list (the reset envs' _compute_observations(env_ids)) and the rollout
// step (progress_buf += 1, the step into experience-buffer slices, dones = float(reset)).
#include <type_traits>

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

enum class ZMode { kStep, kObsList, kRollout };

// A pointer parameter only mode Use reads or writes, __restrict__ in that mode alone: an unused restrict parameter still changes
// which products ptxas contracts into FMAs, and with that the last bit of some SMPL-X observation columns.
template <ZMode Use, ZMode M, class T>
using ModePtr = std::conditional_t<Use == M, T* __restrict__, T*>;

// kObsList: the envs env_list[0 .. *count) (the count read on the device).  kRollout: progress_buf += 1 (humanoid.py:1317) by the lane
// that reads it back in the per-env code, then the step, then the done flag.
template <class L, ZMode M>
__global__ void __launch_bounds__(256) ztask_kernel(const typename L::StepArgs a, ModePtr<ZMode::kObsList, M, const long long> env_list,
                                                    ModePtr<ZMode::kObsList, M, const int> count, ModePtr<ZMode::kRollout, M, float> dones,
                                                    long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long* progress = const_cast<long long*>(reinterpret_cast<const long long*>(a.progress_buf));
  if constexpr (M == ZMode::kObsList) n = *count;
  for (long long i = blockIdx.x * 8ll + warp; i < n; i += 8ll * gridDim.x) {
    const long long e = M == ZMode::kObsList ? env_list[i] : i;
    if constexpr (M == ZMode::kRollout) {
      if (lane == 0) progress[e] += 1;
    }
    ztask_env<L, M == ZMode::kObsList>(a, e, lane);
    if constexpr (M == ZMode::kRollout) {
      if (lane == 0) dones[e] = static_cast<float>(a.reset_buf[e]);
    }
  }
}

// The argument checks of each struct, `who` prefixing the messages.  The list observation reads the observation inputs alone.
int check_step_args(const pulse_reach_step_args_t& a, ZMode mode, const char* who) {
  PULSE_REQUIRE(a.body_state && a.tar_pos && a.obs_buf, "%s: null buffer", who);
  PULSE_REQUIRE(a.body_env_stride >= 24 * 13 && a.obs_stride >= PULSE_REACH_OBS, "%s: bad strides", who);
  if (mode == ZMode::kObsList) return PULSE_OK;
  PULSE_REQUIRE(a.progress_buf && a.rew_buf && a.reset_buf && a.terminate_buf, "%s: null buffer", who);
  PULSE_REQUIRE(a.reach_body_id >= 0 && a.reach_body_id < 24, "%s: reach_body_id out of range", who);
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "%s: termination_heights required", who);
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= 24 * 3, "%s: bad contact stride", who);
  return PULSE_OK;
}

int check_step_args(const pulse_ztask_step_args_t& a, ZMode mode, const char* who) {
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_SPEED || a.kind == PULSE_ZTASK_STRIKE, "%s: unknown task kind %d", who, a.kind);
  const bool speed = a.kind == PULSE_ZTASK_SPEED;
  PULSE_REQUIRE(a.body_state && a.obs_buf, "%s: null buffer", who);
  PULSE_REQUIRE(a.body_env_stride >= 24 * 13, "%s: body_env_stride %lld < 312", who, (long long)a.body_env_stride);
  const int width = speed ? PULSE_SPEED_OBS : PULSE_STRIKE_OBS;
  PULSE_REQUIRE(a.obs_stride >= width, "%s: obs_stride %lld < %d", who, (long long)a.obs_stride, width);
  PULSE_REQUIRE(!speed || a.tar_speed != nullptr, "%s: speed task needs tar_speed", who);
  PULSE_REQUIRE(speed || a.target_states != nullptr, "%s: strike task needs target_states", who);
  if (mode == ZMode::kObsList) {
    PULSE_REQUIRE(speed || a.target_env_stride >= 13, "%s: strike needs target_env_stride >= 13", who);
    return PULSE_OK;
  }
  PULSE_REQUIRE(a.progress_buf && a.prev_root_pos && a.rew_buf && a.reset_buf && a.terminate_buf, "%s: null buffer", who);
  PULSE_REQUIRE(a.dt > 0.0f, "%s: dt must be positive", who);
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "%s: termination_heights required", who);
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= 24 * 3, "%s: bad contact stride", who);
  if (speed) {
    PULSE_REQUIRE(a.dof_force == nullptr || (a.dof_vel != nullptr && a.dof_elem_stride >= 1), "%s: power term needs dof_vel", who);
    PULSE_REQUIRE(a.reward_raw == nullptr || a.raw_stride >= (a.dof_force ? 2 : 1), "%s: raw_stride too small", who);
  } else {
    PULSE_REQUIRE(a.tar_contact_forces != nullptr, "%s: strike task needs tar_contact_forces", who);
  }
  return PULSE_OK;
}

int check_step_args(const pulse_smplx_speed_step_args_t& a, ZMode mode, const char* who) {
  PULSE_REQUIRE(a.body_state && a.obs_buf && a.tar_speed, "%s: null body_state / obs_buf / tar_speed", who);
  PULSE_REQUIRE(a.body_env_stride >= PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W, "%s: body_env_stride %lld < %d", who,
                (long long)a.body_env_stride, PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W);
  PULSE_REQUIRE(a.obs_stride >= PULSE_SMPLX_SPEED_OBS, "%s: obs_stride %lld < %d", who, (long long)a.obs_stride, PULSE_SMPLX_SPEED_OBS);
  if (mode == ZMode::kObsList) return PULSE_OK;
  PULSE_REQUIRE(a.progress_buf && a.prev_root_pos && a.rew_buf && a.reset_buf && a.terminate_buf, "%s: null buffer", who);
  PULSE_REQUIRE(a.dt > 0.0f, "%s: dt must be positive", who);
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "%s: termination_heights required", who);
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= PULSE_SMPLX_BODIES * 3, "%s: contact_env_stride %lld < %d", who,
                (long long)a.contact_env_stride, PULSE_SMPLX_BODIES * 3);
  PULSE_REQUIRE(a.reward_raw == nullptr || a.raw_stride >= 1, "%s: raw_stride too small", who);
  return PULSE_OK;
}

int check_step_args(const pulse_smplx_target_step_args_t& a, ZMode mode, const char* who) {
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
  if (mode == ZMode::kObsList) return PULSE_OK;
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

// Every step entry point: the mode's own pointers, the struct's checks, then one launch (none for an empty list).
template <class L>
int launch_ztask(const typename L::StepArgs* args, ZMode mode, const int64_t* env_list, const int32_t* count, float* dones, int64_t n,
                 void* stream, const char* who) {
  PULSE_REQUIRE(args != nullptr, "%s: null args", who);
  PULSE_REQUIRE(mode != ZMode::kObsList || (env_list && count), "%s: null env_list / count", who);
  PULSE_REQUIRE(mode != ZMode::kRollout || dones != nullptr, "%s: null dones", who);
  const int st = check_step_args(*args, mode, who);
  if (st != PULSE_OK) return st;
  PULSE_REQUIRE(mode == ZMode::kObsList ? n >= 0 : n > 0, "%s: num_envs %lld, must be %s", who, (long long)n,
                mode == ZMode::kObsList ? "non-negative" : "positive");
  if (n == 0) return PULSE_OK;
  const unsigned grid = grid_for(n, 8);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long* list = reinterpret_cast<const long long*>(env_list);
  switch (mode) {
    case ZMode::kStep: ztask_kernel<L, ZMode::kStep><<<grid, 256, 0, s>>>(*args, list, count, dones, n); break;
    case ZMode::kObsList: ztask_kernel<L, ZMode::kObsList><<<grid, 256, 0, s>>>(*args, list, count, dones, n); break;
    case ZMode::kRollout: ztask_kernel<L, ZMode::kRollout><<<grid, 256, 0, s>>>(*args, list, count, dones, n); break;
  }
  PULSE_LAUNCH_OK(who);
  return PULSE_OK;
}

}  // namespace
}  // namespace pulse

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

using pulse::ZMode;
using pulse::launch_ztask;

extern "C" int pulse_reach_step(const pulse_reach_step_args_t* args, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplReachLayout>(args, ZMode::kStep, nullptr, nullptr, nullptr, num_envs, stream, "pulse_reach_step");
}
extern "C" int pulse_reach_obs_list(const pulse_reach_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs,
                                    void* stream) {
  return launch_ztask<pulse::SmplReachLayout>(args, ZMode::kObsList, env_list, count, nullptr, num_envs, stream, "pulse_reach_obs_list");
}
extern "C" int pulse_reach_rollout_step(const pulse_reach_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplReachLayout>(args, ZMode::kRollout, nullptr, nullptr, dones, num_envs, stream, "pulse_reach_rollout_step");
}

extern "C" int pulse_ztask_step(const pulse_ztask_step_args_t* args, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplLayout>(args, ZMode::kStep, nullptr, nullptr, nullptr, num_envs, stream, "pulse_ztask_step");
}
extern "C" int pulse_ztask_obs_list(const pulse_ztask_step_args_t* args, const int64_t* env_list, const int32_t* count, int64_t num_envs,
                                    void* stream) {
  return launch_ztask<pulse::SmplLayout>(args, ZMode::kObsList, env_list, count, nullptr, num_envs, stream, "pulse_ztask_obs_list");
}
extern "C" int pulse_ztask_rollout_step(const pulse_ztask_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplLayout>(args, ZMode::kRollout, nullptr, nullptr, dones, num_envs, stream, "pulse_ztask_rollout_step");
}

extern "C" int pulse_smplx_speed_step(const pulse_smplx_speed_step_args_t* args, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplxLayout>(args, ZMode::kStep, nullptr, nullptr, nullptr, num_envs, stream, "pulse_smplx_speed_step");
}
extern "C" int pulse_smplx_speed_obs_list(const pulse_smplx_speed_step_args_t* args, const int64_t* env_list, const int32_t* count,
                                          int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplxLayout>(args, ZMode::kObsList, env_list, count, nullptr, num_envs, stream, "pulse_smplx_speed_obs_list");
}
extern "C" int pulse_smplx_speed_rollout_step(const pulse_smplx_speed_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplxLayout>(args, ZMode::kRollout, nullptr, nullptr, dones, num_envs, stream, "pulse_smplx_speed_rollout_step");
}

extern "C" int pulse_smplx_target_step(const pulse_smplx_target_step_args_t* args, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplxTargetLayout>(args, ZMode::kStep, nullptr, nullptr, nullptr, num_envs, stream, "pulse_smplx_target_step");
}
extern "C" int pulse_smplx_target_obs_list(const pulse_smplx_target_step_args_t* args, const int64_t* env_list, const int32_t* count,
                                           int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplxTargetLayout>(args, ZMode::kObsList, env_list, count, nullptr, num_envs, stream,
                                                "pulse_smplx_target_obs_list");
}
extern "C" int pulse_smplx_target_rollout_step(const pulse_smplx_target_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  return launch_ztask<pulse::SmplxTargetLayout>(args, ZMode::kRollout, nullptr, nullptr, dones, num_envs, stream,
                                                "pulse_smplx_target_rollout_step");
}
