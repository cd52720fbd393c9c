// Per-step env reset on the device, no host synchronisation (SURVEY rows a13 / 8f-3):
//   reset_compact_kernel    reset_buf != 0 (or an explicit id list) -> ascending env list + actor-id list + device-side count
//                           (what `nonzero` + `_humanoid_actor_ids[env_ids]` produce in the reference, humanoid.py:589-593,
//                           amp_agent.py:413-416) -- one CTA, ballot / prefix scan, no atomics (the order is deterministic);
//   reset_ref_state_kernel  (reset_state.cuh) the start-time draw, MotionLib gather, scatter into the simulator's views and the
//                           AMP back-fill of every env in that list.
#include "reset_state.cuh"

namespace pulse {
namespace {

__global__ void __launch_bounds__(kCompactThreads) reset_compact_kernel(const pulse_reset_args_t a, long long num_envs) {
  __shared__ int warp_cnt[kCompactThreads / 32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const long long n = a.env_ids_in != nullptr ? a.num_ids : num_envs;
  for (long long c0 = 0; c0 < n; c0 += kCompactThreads) {
    const long long env = reset_candidate(a, c0 + threadIdx.x, n);
    const int pos = compact_slot(env >= 0, warp_cnt, &base);
    if (pos >= 0) {
      a.env_list[pos] = env;
      if (a.actor_list != nullptr) a.actor_list[pos] = a.actor_ids != nullptr ? a.actor_ids[env] : static_cast<int>(env);
    }
  }
  if (threadIdx.x == 0) *a.count = base;
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_reset_ref_state(const pulse_motionlib_t* lib, const pulse_reset_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "pulse_reset_ref_state: null lib/args");
  const pulse_reset_args_t& a = *args;
  const int rc = check_ref_state_args(lib, a, num_envs, "pulse_reset_ref_state");
  if (rc != PULSE_OK) return rc;
  if (num_envs == 0) return PULSE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  reset_compact_kernel<<<1, kCompactThreads, 0, st>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("reset_compact_kernel");
  return launch_ref_state(lib, a, a.env_ids_in != nullptr ? a.num_ids : num_envs, st);
}
