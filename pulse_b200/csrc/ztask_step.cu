// Post-physics step of the downstream latent-space tasks HumanoidReach (SURVEY K21), HumanoidSpeedZ and HumanoidStrikeZ (SURVEY 8f-4):
// one warp per env, lane = body -- self observation (humanoid.py:1675-1731), task observation, reward and reset in one launch.
//   reach   compute_location_observations / compute_reach_reward  phc/env/tasks/humanoid_reach.py:224-250, target resampling
//           (_update_task :126-147) in reach_update_task_kernel, reset = compute_humanoid_reset  humanoid.py:1573-1608
//   speed   compute_speed_observations / compute_speed_reward   phc/env/tasks/humanoid_speed.py:310-343, power term :215-222,
//           reset = compute_humanoid_reset
//   strike  compute_strike_observations / compute_strike_reward  phc/env/tasks/humanoid_strike.py:270-328,
//           reset = the strike variant of compute_humanoid_reset  :330-375
#include "humanoid_obs.cuh"

namespace pulse {
namespace {

constexpr int kZB = PULSE_NUM_BODIES;

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

// One env of the reach step, lane = body.  kObsOnly: the observation alone (the reset envs' _compute_observations(env_ids)).
template <bool kObsOnly>
__device__ __forceinline__ void reach_env(const pulse_reach_step_args_t& a, long long e, int lane) {
  const int j = lane;
  const bool body = j < kZB;
  const float* bs = a.body_state + e * a.body_env_stride + (body ? j : 0) * 13;
  Vec3 p = {bs[0], bs[1], bs[2]}, v = {bs[7], bs[8], bs[9]}, w = {bs[10], bs[11], bs[12]};
  Quat q = {bs[3], bs[4], bs[5], bs[6]};
  const Vec3 p_root = {__shfl_sync(kFull, p.x, 0), __shfl_sync(kFull, p.y, 0), __shfl_sync(kFull, p.z, 0)};
  const Quat q_root = {__shfl_sync(kFull, q.x, 0), __shfl_sync(kFull, q.y, 0), __shfl_sync(kFull, q.z, 0), __shfl_sync(kFull, q.w, 0)};
  float hs, hc;
  heading_half(q_root, hs, hc);
  const Yaw yr = make_yaw(Quat{0.0f, 0.0f, -hs, hc});
  float* o = a.obs_buf + e * a.obs_stride;
  if (body) {  // store_self_obs's layout written out, for the reason given in im_step.cu
    if (j == 0) o[0] = p_root.z;
    else {
      const Vec3 lp = yaw_rot(yr, p - p_root);
      o[1 + 3 * (j - 1)] = lp.x; o[2 + 3 * (j - 1)] = lp.y; o[3 + 3 * (j - 1)] = lp.z;
    }
    float six[6];
    qsix(yaw_mul_left(-hs, hc, q), six);
#pragma unroll
    for (int i = 0; i < 6; ++i) o[70 + 6 * j + i] = six[i];
    const Vec3 lv = yaw_rot(yr, v), lw = yaw_rot(yr, w);
    o[214 + 3 * j] = lv.x; o[215 + 3 * j] = lv.y; o[216 + 3 * j] = lv.z;
    o[286 + 3 * j] = lw.x; o[287 + 3 * j] = lw.y; o[288 + 3 * j] = lw.z;
  }
  const Vec3 tar = {a.tar_pos[3 * e], a.tar_pos[3 * e + 1], a.tar_pos[3 * e + 2]};
  const FallFlags fall = fall_flags(a, e, j, body, p.z);
  const bool any_contact = __any_sync(kFull, fall.contact), any_height = __any_sync(kFull, fall.height);
  // the reach body's position, broadcast
  const int rb = a.reach_body_id;
  const Vec3 pr = {__shfl_sync(kFull, p.x, rb), __shfl_sync(kFull, p.y, rb), __shfl_sync(kFull, p.z, rb)};
  if (lane == 0) {
    const Vec3 lt = yaw_rot(yr, tar - p_root);  // compute_location_observations (humanoid_reach.py:224-236)
    o[PULSE_SELF_OBS + 0] = lt.x; o[PULSE_SELF_OBS + 1] = lt.y; o[PULSE_SELF_OBS + 2] = lt.z;
    if constexpr (!kObsOnly) {
      const Vec3 d = tar - pr;                  // compute_reach_reward (:238-250)
      a.rew_buf[e] = expf(-4.0f * (d.x * d.x + d.y * d.y + d.z * d.z));
      const long long prog = a.progress_buf[e];
      const long long term = (any_contact && any_height && prog > 1) ? 1 : 0;
      a.terminate_buf[e] = term;
      a.reset_buf[e] = prog >= a.max_episode_length - 1 ? 1 : term;
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

// One env of the speed / strike step, lane = body.  kObsOnly: the observation alone.
template <bool kObsOnly>
__device__ __forceinline__ void ztask_env(const pulse_ztask_step_args_t& a, long long e, int lane) {
  const int j = lane;
  const bool body = j < kZB;
  const float* bs = a.body_state + e * a.body_env_stride + (body ? j : 0) * 13;
  const Vec3 p = {bs[0], bs[1], bs[2]}, v = {bs[7], bs[8], bs[9]}, w = {bs[10], bs[11], bs[12]};
  const Quat q = {bs[3], bs[4], bs[5], bs[6]};
  const Vec3 p_root = {__shfl_sync(kFull, p.x, 0), __shfl_sync(kFull, p.y, 0), __shfl_sync(kFull, p.z, 0)};
  const Quat q_root = {__shfl_sync(kFull, q.x, 0), __shfl_sync(kFull, q.y, 0), __shfl_sync(kFull, q.z, 0), __shfl_sync(kFull, q.w, 0)};
  float hs, hc;
  heading_half(q_root, hs, hc);
  const Yaw yr = make_yaw(Quat{0.0f, 0.0f, -hs, hc});
  float* o = a.obs_buf + e * a.obs_stride;
  if (body) store_self_obs(o, j, p, p_root, q, v, w, hs, hc, yr);
  const FallFlags fall = fall_flags(a, e, j, body, p.z);
  // strike: a body that is neither a ground-contact body nor a strike body pressing harder than 50 N (humanoid_strike.py:356-364)
  bool hard_contact = false;
  if (a.enable_early_termination && body && a.contact_forces != nullptr && !(((a.contact_body_mask | a.strike_body_mask) >> j) & 1u)) {
    const float* cf = a.contact_forces + e * a.contact_env_stride + j * 3;
    hard_contact = fabsf(cf[0]) > 50.0f || fabsf(cf[1]) > 50.0f || fabsf(cf[2]) > 50.0f;
  }
  const bool any_contact = __any_sync(kFull, fall.contact), any_height = __any_sync(kFull, fall.height);
  const bool any_hard = __any_sync(kFull, hard_contact);
  // power term of the speed task: -c * sum |tau * qdot|, zero for progress <= 3 (humanoid_speed.py:215-222)
  const float power = a.kind == PULSE_ZTASK_SPEED && a.dof_force != nullptr ? dof_power(a, e, lane) : 0.0f;
  if (lane == 0) {
    const long long prog = a.progress_buf[e];
    const float* pr = a.prev_root_pos + 3 * e;
    const float vx = (p_root.x - pr[0]) / a.dt, vy = (p_root.y - pr[1]) / a.dt;   // root_vel = delta_root_pos / dt
    float* t = o + PULSE_SELF_OBS;
    bool failed = any_contact && any_height;
    if (a.kind == PULSE_ZTASK_SPEED) {
      // observation: heading-frame x axis (first two components) and the target speed (:310-325)
      const Vec3 d = yaw_rot(yr, Vec3{1.0f, 0.0f, 0.0f});
      const float ts = a.tar_speed[e];
      t[0] = d.x; t[1] = d.y; t[2] = ts;
      if constexpr (kObsOnly) return;
      const float err = ts - vx;
      float rew = expf(-0.25f * (err * err + 0.1f * vy * vy));                    // :327-343
      if (a.reward_raw != nullptr) a.reward_raw[e * a.raw_stride] = rew;
      if (a.dof_force != nullptr) {
        const float pw = prog <= 3 ? 0.0f : -a.power_coefficient * power;
        rew += pw;
        if (a.reward_raw != nullptr) a.reward_raw[e * a.raw_stride + 1] = pw;
      }
      a.rew_buf[e] = rew;
    } else {
      const float* ts = a.target_states + e * a.target_env_stride;
      const Vec3 tp = {ts[0], ts[1], ts[2]};
      const Quat tq = {ts[3], ts[4], ts[5], ts[6]};
      // observation (:270-293): target position relative to the root with the ABSOLUTE height, 6D rotation, velocities, heading frame
      const Vec3 lp = yaw_rot(yr, Vec3{tp.x - p_root.x, tp.y - p_root.y, tp.z});
      t[0] = lp.x; t[1] = lp.y; t[2] = lp.z;
      qsix(yaw_mul_left(-hs, hc, tq), t + 3);
      const Vec3 lv = yaw_rot(yr, Vec3{ts[7], ts[8], ts[9]}), lw = yaw_rot(yr, Vec3{ts[10], ts[11], ts[12]});
      t[9] = lv.x; t[10] = lv.y; t[11] = lv.z;
      t[12] = lw.x; t[13] = lw.y; t[14] = lw.z;
      if constexpr (kObsOnly) return;
      // reward (:295-328)
      const float rot_err = 2.0f * tq.w * tq.w - 1.0f + 2.0f * tq.z * tq.z;      // z component of quat_rotate(tar_rot, [0, 0, 1])
      const float rot_r = fmaxf(1.0f - rot_err, 0.0f);
      float dx = tp.x - p_root.x, dy = tp.y - p_root.y;
      const float dn = fmaxf(sqrtf(dx * dx + dy * dy), 1e-12f);                    // torch.nn.functional.normalize (eps 1e-12)
      dx /= dn; dy /= dn;
      const float dir_speed = dx * vx + dy * vy;
      const float verr = fmaxf(1.0f - dir_speed, 0.0f);
      float vel_r = expf(-4.0f * verr * verr);
      if (dir_speed <= 0.0f) vel_r = 0.0f;
      float rew = 0.6f * rot_r + 0.4f * vel_r;
      if (rot_err < 0.2f) rew = 1.0f;
      a.rew_buf[e] = rew;
      // reset (:330-375): also fails when the target is pushed (> 50 N horizontally) while a non-strike body presses hard
      const float* tc = a.tar_contact_forces + e * a.tar_contact_env_stride;
      const bool tar_contact = fabsf(tc[0]) > 50.0f || fabsf(tc[1]) > 50.0f;
      failed = failed || (a.enable_early_termination && tar_contact && any_hard);
    }
    const long long term = (a.enable_early_termination && failed && prog > 1) ? 1 : 0;
    a.terminate_buf[e] = term;
    a.reset_buf[e] = prog >= a.max_episode_length - 1 ? 1 : term;
  }
}

__global__ void __launch_bounds__(256) ztask_step_kernel(const pulse_ztask_step_args_t a, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long e = blockIdx.x * 8ll + warp; e < n; e += 8ll * gridDim.x) ztask_env<false>(a, e, lane);
}

__global__ void __launch_bounds__(256) ztask_obs_list_kernel(const pulse_ztask_step_args_t a, const long long* __restrict__ env_list,
                                                             const int* __restrict__ count) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = *count;
  for (long long i = blockIdx.x * 8ll + warp; i < n; i += 8ll * gridDim.x) ztask_env<true>(a, env_list[i], lane);
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
  ztask_step_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)num_envs);
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
  ztask_obs_list_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, reinterpret_cast<const long long*>(env_list), count);
  PULSE_LAUNCH_OK("ztask_obs_list_kernel");
  return PULSE_OK;
}
