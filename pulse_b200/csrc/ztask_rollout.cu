// Rollout glue of the latent-space tasks HumanoidReachZ / HumanoidSpeedZ / HumanoidStrikeZ (AMPAgent.play_steps, amp_agent.py:341-439;
// HumanoidZ.step -> step_z, humanoid_z.py:157-173), every kernel writing into experience-buffer slices (pointer + stride):
//   latent_post_kernel        the latent policy's sampling (policy_post_kernel's draws and arithmetic), neglogp, the de-normalised value
//                             and z = prior_mu + a_z as bf16 into the decoder operand: pulse_policy_post + pulse_vae_reparam in one launch;
//   ztask_pre_physics_kernel  PD targets from the decoder output, prev_root_pos, and _update_task of the due envs with draws injected or
//                             made here (Philox index plane e + 3 * 2^32);
//   reach_rollout_kernel /    progress_buf += 1, then the per-env step code of ztask_env.cuh into the next step's observation slice and
//   ztask_rollout_kernel      the step's reward row, then dones = float(reset); ztask_rollout_kernel<SmplxLayout> is the SMPL-X
//                             speed task's (pulse_smplx_speed_rollout_step), ztask_rollout_kernel<SmplxTargetLayout> the SMPL-X
//                             reach and strike tasks' (pulse_smplx_target_rollout_step).
// The entry points, argument structs and the Philox word layout are documented in include/pulse_b200.h.
#include <cuda_bf16.h>

#include "philox.cuh"
#include "value_unnorm.cuh"
#include "ztask_env.cuh"

namespace pulse {
namespace {

constexpr unsigned long long kUpdateStream = 3ull << 32;   // Philox index e + 3 * 2^32: _update_task draws

__global__ void __launch_bounds__(128) latent_post_kernel(const pulse_latent_post_args_t a, long long rows) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int A = a.latent;
  const unsigned long long off = a.rng_offset != nullptr ? *a.rng_offset + a.rng_step : a.rng_step;
  __nv_bfloat16* zb = reinterpret_cast<__nv_bfloat16*>(a.z_bf16);
  float acc = 0.0f, ls = 0.0f;
  // lanes take PAIRS of latent dimensions (2*lane + 64*i), the indexing and arithmetic of policy_post_kernel
  for (int i = 0; 2 * lane + 64 * i < A; ++i) {
    const int k0 = 2 * lane + 64 * i;
    float e0, e1;
    if (a.eps != nullptr) {
      e0 = a.eps[row * a.ld_eps + k0];
      e1 = k0 + 1 < A ? a.eps[row * a.ld_eps + k0 + 1] : 0.0f;
    } else {
      const Philox4 r = philox4x32_10(a.seed, static_cast<unsigned long long>(row) * 64ull + static_cast<unsigned long long>(lane + 32 * i), off);
      box_muller(r.x, r.y, e0, e1);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = k0 + h;
      if (k >= A) break;
      const float l = a.logstd[k];
      const float sg = expf(l);
      const float m = a.mu[row * a.ld_mu + k];
      const float act = m + sg * (h == 0 ? e0 : e1);
      a.actions[row * a.ld_actions + k] = act;
      zb[row * a.ld_z + k] = __float2bfloat16(__fadd_rn(a.prior_mu[row * a.ld_prior + k], act));   // humanoid_z.py:104-107
      const float z = (act - m) / sg;
      acc += z * z;
      ls += l;
    }
  }
  acc = warp_sum(acc);
  ls = warp_sum(ls);
  if (lane == 0) {
    a.neglogp[row * a.ld_neglogp] = 0.5f * acc + 0.5f * 1.8378770664093453f * A + ls;   // log(2*pi)
    a.values_out[row * a.ld_values] = value_unnorm(a.value[row * a.ld_value], a.value_mean, a.value_var, a.value_eps);
  }
}

__global__ void __launch_bounds__(256) ztask_pre_physics_kernel(const pulse_ztask_pre_physics_args_t a, long long n) {
  const int dofs = a.dofs;
  const long long total = n * dofs;
  const unsigned long long off = a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull);
  const unsigned long long span = static_cast<unsigned long long>(a.steps_max - a.steps_min);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long e = i / dofs;
    const int d = static_cast<int>(i - e * dofs);
    const float v = __fadd_rn(a.pd_offset[d], __fmul_rn(a.pd_scale[d], a.action[e * a.ld_action + d]));   // pd_targets_kernel's two roundings
    a.pd_out[e * a.ld_pd + d] = (a.freeze != nullptr && a.freeze[d]) ? 0.0f : v;
    if (d < 3 && a.prev_root_pos != nullptr) a.prev_root_pos[3 * e + d] = a.root_states[e * a.root_env_stride + d];
    if (d != 0 || a.kind == PULSE_ZTASK_STRIKE) continue;
    const long long prog = a.progress_buf[e];
    if (prog < a.change_steps[e]) continue;
    Philox4 r{0u, 0u, 0u, 0u};
    if (a.rand == nullptr || a.steps_in == nullptr) r = philox4x32_10(a.seed, static_cast<unsigned long long>(e) + kUpdateStream, off);
    const long long steps = a.steps_in != nullptr ? a.steps_in[e] : a.steps_min + static_cast<long long>((static_cast<unsigned long long>(r.w) * span) >> 32);
    if (a.kind == PULSE_ZTASK_REACH) {   // reach_update_task_kernel's expressions
      const float u0 = a.rand ? a.rand[3 * e] : u01(r.x), u1 = a.rand ? a.rand[3 * e + 1] : u01(r.y), u2 = a.rand ? a.rand[3 * e + 2] : u01(r.z);
      a.tar_pos[3 * e + 0] = a.dist_max * (2.0f * u0 - 1.0f);
      a.tar_pos[3 * e + 1] = a.dist_max * (2.0f * u1 - 1.0f);
      a.tar_pos[3 * e + 2] = (a.height_max - a.height_min) * u2 + a.height_min;
    } else {                             // humanoid_speed.py:166-175
      const float u = a.rand ? a.rand[e] : u01(r.x);
      a.tar_speed[e] = __fadd_rn(__fmul_rn(a.speed_scale, u), a.speed_min);
    }
    a.change_steps[e] = prog + steps;
  }
}

// progress_buf += 1 (humanoid.py:1317) by the lane that reads it back in the per-env code, then the step, then the done flag.
__global__ void __launch_bounds__(256) reach_rollout_kernel(const pulse_reach_step_args_t a, float* __restrict__ dones, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long* progress = const_cast<long long*>(reinterpret_cast<const long long*>(a.progress_buf));
  for (long long e = blockIdx.x * 8ll + warp; e < n; e += 8ll * gridDim.x) {
    if (lane == 0) progress[e] += 1;
    reach_env<false>(a, e, lane);
    if (lane == 0) dones[e] = static_cast<float>(a.reset_buf[e]);
  }
}

template <class L>
__global__ void __launch_bounds__(256) ztask_rollout_kernel(const typename L::StepArgs a, float* __restrict__ dones, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long* progress = const_cast<long long*>(reinterpret_cast<const long long*>(a.progress_buf));
  for (long long e = blockIdx.x * 8ll + warp; e < n; e += 8ll * gridDim.x) {
    if (lane == 0) progress[e] += 1;
    ztask_env<L, false>(a, e, lane);
    if (lane == 0) dones[e] = static_cast<float>(a.reset_buf[e]);
  }
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_latent_post(const pulse_latent_post_args_t* args, int64_t rows, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_latent_post: null args");
  PULSE_REQUIRE(rows >= 0, "pulse_latent_post: negative rows");
  const pulse_latent_post_args_t& a = *args;
  PULSE_REQUIRE(a.mu && a.logstd && a.actions && a.neglogp, "pulse_latent_post: null mu / logstd / actions / neglogp");
  PULSE_REQUIRE(a.value && a.values_out && a.prior_mu && a.z_bf16, "pulse_latent_post: null value / values_out / prior_mu / z_bf16");
  PULSE_REQUIRE(a.latent >= 1 && a.latent <= 128, "pulse_latent_post: latent %d outside [1,128]", a.latent);
  PULSE_REQUIRE(a.ld_mu >= a.latent && a.ld_actions >= a.latent && a.ld_prior >= a.latent && a.ld_z >= a.latent && a.ld_neglogp >= 1 &&
                    a.ld_value >= 1 && a.ld_values >= 1, "pulse_latent_post: leading dimensions too small");
  PULSE_REQUIRE(a.eps == nullptr || a.ld_eps >= a.latent, "pulse_latent_post: ld_eps too small");
  PULSE_REQUIRE((a.value_mean == nullptr) == (a.value_var == nullptr), "pulse_latent_post: value_mean and value_var go together");
  if (rows == 0) return PULSE_OK;
  latent_post_kernel<<<static_cast<unsigned>((rows * 32 + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)rows);
  PULSE_LAUNCH_OK("latent_post_kernel");
  return PULSE_OK;
}

extern "C" int pulse_ztask_pre_physics(const pulse_ztask_pre_physics_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_ztask_pre_physics: null args");
  const pulse_ztask_pre_physics_args_t& a = *args;
  PULSE_REQUIRE(num_envs >= 0 && num_envs < (1ll << 31), "pulse_ztask_pre_physics: num_envs %lld outside [0, 2^31)", (long long)num_envs);
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_REACH || a.kind == PULSE_ZTASK_SPEED || a.kind == PULSE_ZTASK_STRIKE,
                "pulse_ztask_pre_physics: unknown task kind %d", a.kind);
  PULSE_REQUIRE(a.action && a.pd_offset && a.pd_scale && a.pd_out, "pulse_ztask_pre_physics: null action / pd_offset / pd_scale / pd_out");
  PULSE_REQUIRE(a.dofs >= 3 && a.ld_action >= a.dofs && a.ld_pd >= a.dofs, "pulse_ztask_pre_physics: dofs %d < 3 or row strides too small", a.dofs);
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_REACH || (a.root_states && a.prev_root_pos && a.root_env_stride >= 3),
                "pulse_ztask_pre_physics: the speed and strike tasks need root_states and prev_root_pos");
  PULSE_REQUIRE(a.prev_root_pos == nullptr || (a.root_states != nullptr && a.root_env_stride >= 3), "pulse_ztask_pre_physics: prev_root_pos needs root_states");
  if (a.kind != PULSE_ZTASK_STRIKE) {
    PULSE_REQUIRE(a.progress_buf && a.change_steps, "pulse_ztask_pre_physics: null progress_buf / change_steps");
    PULSE_REQUIRE(a.kind != PULSE_ZTASK_REACH || a.tar_pos != nullptr, "pulse_ztask_pre_physics: the reach task needs tar_pos");
    PULSE_REQUIRE(a.kind != PULSE_ZTASK_SPEED || a.tar_speed != nullptr, "pulse_ztask_pre_physics: the speed task needs tar_speed");
    PULSE_REQUIRE(a.steps_in != nullptr || a.steps_max > a.steps_min, "pulse_ztask_pre_physics: empty randint range [%lld, %lld)",
                  (long long)a.steps_min, (long long)a.steps_max);
  }
  if (num_envs == 0) return PULSE_OK;
  ztask_pre_physics_kernel<<<grid_for(num_envs * a.dofs, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("ztask_pre_physics_kernel");
  return PULSE_OK;
}

extern "C" int pulse_reach_rollout_step(const pulse_reach_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args && dones, "pulse_reach_rollout_step: null args / dones");
  const pulse_reach_step_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.tar_pos && a.progress_buf && a.obs_buf && a.rew_buf && a.reset_buf && a.terminate_buf,
                "pulse_reach_rollout_step: null buffer");
  PULSE_REQUIRE(num_envs > 0 && a.body_env_stride >= 24 * 13 && a.obs_stride >= PULSE_REACH_OBS, "pulse_reach_rollout_step: bad strides");
  PULSE_REQUIRE(a.reach_body_id >= 0 && a.reach_body_id < 24, "pulse_reach_rollout_step: reach_body_id out of range");
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "pulse_reach_rollout_step: termination_heights required");
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= 24 * 3, "pulse_reach_rollout_step: bad contact stride");
  reach_rollout_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, dones, (long long)num_envs);
  PULSE_LAUNCH_OK("reach_rollout_kernel");
  return PULSE_OK;
}

extern "C" int pulse_ztask_rollout_step(const pulse_ztask_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args && dones, "pulse_ztask_rollout_step: null args / dones");
  const pulse_ztask_step_args_t& a = *args;
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_SPEED || a.kind == PULSE_ZTASK_STRIKE, "pulse_ztask_rollout_step: unknown task kind %d", a.kind);
  PULSE_REQUIRE(num_envs > 0, "pulse_ztask_rollout_step: num_envs must be positive");
  PULSE_REQUIRE(a.body_state && a.progress_buf && a.prev_root_pos && a.obs_buf && a.rew_buf && a.reset_buf && a.terminate_buf,
                "pulse_ztask_rollout_step: null buffer");
  PULSE_REQUIRE(a.dt > 0.0f, "pulse_ztask_rollout_step: dt must be positive");
  PULSE_REQUIRE(a.body_env_stride >= 24 * 13, "pulse_ztask_rollout_step: body_env_stride %lld < 312", (long long)a.body_env_stride);
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "pulse_ztask_rollout_step: termination_heights required");
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= 24 * 3, "pulse_ztask_rollout_step: bad contact stride");
  if (a.kind == PULSE_ZTASK_SPEED) {
    PULSE_REQUIRE(a.tar_speed != nullptr, "pulse_ztask_rollout_step: speed task needs tar_speed");
    PULSE_REQUIRE(a.obs_stride >= PULSE_SPEED_OBS, "pulse_ztask_rollout_step: obs_stride %lld < %d", (long long)a.obs_stride, PULSE_SPEED_OBS);
    PULSE_REQUIRE(a.dof_force == nullptr || (a.dof_vel != nullptr && a.dof_elem_stride >= 1), "pulse_ztask_rollout_step: power term needs dof_vel");
    PULSE_REQUIRE(a.reward_raw == nullptr || a.raw_stride >= (a.dof_force ? 2 : 1), "pulse_ztask_rollout_step: raw_stride too small");
  } else {
    PULSE_REQUIRE(a.target_states && a.tar_contact_forces, "pulse_ztask_rollout_step: strike task needs target_states and tar_contact_forces");
    PULSE_REQUIRE(a.obs_stride >= PULSE_STRIKE_OBS, "pulse_ztask_rollout_step: obs_stride %lld < %d", (long long)a.obs_stride, PULSE_STRIKE_OBS);
  }
  ztask_rollout_kernel<SmplLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, dones, (long long)num_envs);
  PULSE_LAUNCH_OK("ztask_rollout_kernel");
  return PULSE_OK;
}

namespace pulse {
int check_smplx_speed_args(const pulse_smplx_speed_step_args_t* args, bool step, const char* who);   // ztask_step.cu
}  // namespace pulse

extern "C" int pulse_smplx_speed_rollout_step(const pulse_smplx_speed_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  using namespace pulse;
  const int st = check_smplx_speed_args(args, true, "pulse_smplx_speed_rollout_step");
  if (st != PULSE_OK) return st;
  PULSE_REQUIRE(dones != nullptr, "pulse_smplx_speed_rollout_step: null dones");
  PULSE_REQUIRE(num_envs > 0, "pulse_smplx_speed_rollout_step: num_envs must be positive");
  ztask_rollout_kernel<SmplxLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, dones, (long long)num_envs);
  PULSE_LAUNCH_OK("ztask_rollout_kernel<SmplxLayout>");
  return PULSE_OK;
}

namespace pulse {
int check_smplx_target_args(const pulse_smplx_target_step_args_t* args, bool step, const char* who);   // ztask_step.cu
}  // namespace pulse

extern "C" int pulse_smplx_target_rollout_step(const pulse_smplx_target_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  using namespace pulse;
  const int st = check_smplx_target_args(args, true, "pulse_smplx_target_rollout_step");
  if (st != PULSE_OK) return st;
  PULSE_REQUIRE(dones != nullptr, "pulse_smplx_target_rollout_step: null dones");
  PULSE_REQUIRE(num_envs > 0, "pulse_smplx_target_rollout_step: num_envs must be positive");
  ztask_rollout_kernel<SmplxTargetLayout><<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(*args, dones, (long long)num_envs);
  PULSE_LAUNCH_OK("ztask_rollout_kernel<SmplxTargetLayout>");
  return PULSE_OK;
}
