// Rollout glue of the latent-space tasks HumanoidReachZ / HumanoidSpeedZ / HumanoidStrikeZ (AMPAgent.play_steps, amp_agent.py:341-439;
// HumanoidZ.step -> step_z, humanoid_z.py:157-173), every kernel writing into experience-buffer slices (pointer + stride):
//   latent_post_kernel        the latent policy's sampling (policy_post_kernel's draws and arithmetic), neglogp, the de-normalised value
//                             and z = prior_mu + a_z as bf16 into the decoder operand: pulse_policy_post + pulse_vae_reparam in one launch;
//   ztask_pre_physics_kernel  PD targets from the decoder output, prev_root_pos, and _update_task of the due envs with draws injected or
//                             made here (Philox index plane e + 3 * 2^32).
// The rollout step kernels (progress_buf += 1, the step into the experience-buffer slices, dones = float(reset)) are ztask_step.cu's
// ztask_kernel in its rollout mode.
// The entry points, argument structs and the Philox word layout are documented in include/pulse_b200.h.
#include <cuda_bf16.h>

#include "philox.cuh"
#include "pulse_common.cuh"
#include "value_unnorm.cuh"

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
