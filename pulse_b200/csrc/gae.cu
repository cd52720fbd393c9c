// GAE / return scan over the rollout buffer and advantage normalisation.
// common_agent.py:493-505 (discount_values), amp_agent.py:427 (returns = advs + values),
// common_agent.py:589-599 (_calc_advs).
//
// T (horizon, 32) is tiny and the scan is sequential in t, so the parallel axis is the env axis:
// one thread per env walks t = T-1 .. 0; the [T,N] inputs are read coalesced across the warp.
// Outputs are transposed to the env-major [N,T] minibatch layout through a padded shared tile so
// both sides stay coalesced.  HBM-bound: 4 reads + 2 writes of 4 B per (t, env).
#include "pulse_common.cuh"

namespace pulse {
namespace {

constexpr int kEnvsPerCta = 32;   // one warp of scanners ...
constexpr int kMaxT = 64;

__global__ void __launch_bounds__(kEnvsPerCta) gae_kernel(const pulse_gae_args_t a, int T, long long n) {
  __shared__ float s_adv[kEnvsPerCta][kMaxT + 1];
  __shared__ float s_ret[kEnvsPerCta][kMaxT + 1];
  const int lane = threadIdx.x;
  const long long e0 = (long long)blockIdx.x * kEnvsPerCta;
  const long long e = e0 + lane;
  float last = 0.0f;
  double sum = 0.0, sq = 0.0;
  if (e < n) {
    for (int t = T - 1; t >= 0; --t) {
      const long long i = (long long)t * n + e;
      const float not_done = 1.0f - a.fdones[i];
      // delta = r + gamma*V' - V ; last = delta + gamma*tau*not_done*last   (reference op order)
      const float delta = __fsub_rn(__fadd_rn(a.rewards[i], __fmul_rn(a.gamma, a.next_values[i])), a.values[i]);
      last = __fadd_rn(delta, __fmul_rn(__fmul_rn(__fmul_rn(a.gamma, a.tau), not_done), last));
      s_adv[lane][t] = last;
      s_ret[lane][t] = __fadd_rn(last, a.values[i]);
      sum += last;
      sq += (double)last * (double)last;
    }
  }
  __syncwarp();
  // env-major write-out: this CTA owns rows e0 .. e0+31, i.e. one contiguous [32*T] span
  const long long rows = (n - e0 < kEnvsPerCta) ? (n - e0) : kEnvsPerCta;
  for (long long k = lane; k < rows * T; k += kEnvsPerCta) {
    const int r = static_cast<int>(k / T), t = static_cast<int>(k % T);
    a.advantages[e0 * T + k] = s_adv[r][t];
    a.returns[e0 * T + k] = s_ret[r][t];
  }
  if (a.adv_sum != nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sum += __shfl_xor_sync(kFull, sum, o);
      sq += __shfl_xor_sync(kFull, sq, o);
    }
    if (lane == 0) {
      atomicAdd(a.adv_sum + 0, sum);
      atomicAdd(a.adv_sum + 1, sq);
    }
  }
}

__global__ void normalize_adv_kernel(float* adv, const double* stats, long long count) {
  const double mean = stats[0] / (double)count;
  double var = (stats[1] - (double)count * mean * mean) / (double)(count - 1);  // unbiased, torch.std default
  if (var < 0.0) var = 0.0;
  const float fmean = (float)mean;
  const float denom = (float)sqrt(var) + 1e-8f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
    adv[i] = (adv[i] - fmean) / denom;
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_gae(const pulse_gae_args_t* args, int32_t horizon, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_gae: null args");
  PULSE_REQUIRE(horizon >= 1 && horizon <= kMaxT, "pulse_gae: horizon %d outside [1,%d]", horizon, kMaxT);
  PULSE_REQUIRE(num_envs >= 0, "pulse_gae: negative num_envs");
  if (num_envs == 0) return PULSE_OK;
  const pulse_gae_args_t& a = *args;
  PULSE_REQUIRE(a.rewards && a.values && a.next_values && a.fdones && a.advantages && a.returns, "pulse_gae: null buffer");
  const unsigned grid = static_cast<unsigned>((num_envs + kEnvsPerCta - 1) / kEnvsPerCta);
  gae_kernel<<<grid, kEnvsPerCta, 0, static_cast<cudaStream_t>(stream)>>>(a, horizon, (long long)num_envs);
  PULSE_LAUNCH_OK("gae_kernel");
  return PULSE_OK;
}

extern "C" int pulse_normalize_advantages(float* advantages, const double* adv_sum, int64_t count, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(advantages && adv_sum, "pulse_normalize_advantages: null buffer");
  PULSE_REQUIRE(count >= 2, "pulse_normalize_advantages: need at least 2 samples");
  normalize_adv_kernel<<<grid_for(count, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(advantages, adv_sum, (long long)count);
  PULSE_LAUNCH_OK("normalize_adv_kernel");
  return PULSE_OK;
}
