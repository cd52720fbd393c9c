// AMP observation (196 floats) + in-place history shift of the [N, steps, 196] buffer.
// humanoid_amp.py:622-630 (_update_hist_amp_obs), :632-667 (_compute_amp_observations),
// :924-969 (build_amp_observations_smpl), humanoid.py:1436-1446 (dof_to_obs_smpl).
//
// One warp per env.  The shift reads the (steps-1) older rows into registers before any store, so
// the in-place move is safe; lanes 0..18 then convert the 19 kept joints' exponential maps to 6-D
// rotations.  Layout of one step: [h | six(hinv*q0) | R v0 | R w0 | 19x six(dof) | 57 dof_vel | 4x R(key-p0)].
#include "humanoid_obs.cuh"

namespace pulse {
namespace {

constexpr int kAmp = PULSE_AMP_OBS;
constexpr int kMaxHist = 16;  // numAMPObsSteps - 1 <= 15

__global__ void __launch_bounds__(128) amp_obs_kernel(const pulse_amp_obs_args_t a, long long n) {
  const long long e = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= n) return;
  float* buf = a.amp_obs_buf + e * (long long)a.num_steps * kAmp;
  const int hist = (a.num_steps - 1) * kAmp;  // floats to move
  // ---- history shift: buf[196 + k] <- buf[k], k < hist; all loads before all stores -------------
  if (a.shift_history && hist > 0) {
    float4 regs[kMaxHist];
    const float4* src = reinterpret_cast<const float4*>(buf);  // rows are 784 B: 16-byte aligned
    const int nvec = hist / 4;                                   // 196 % 4 == 0
#pragma unroll
    for (int i = 0; i < kMaxHist; ++i) {
      int c = lane + 32 * i;
      if (c < nvec) regs[i] = src[c];
    }
    __syncwarp();
    float4* dst = reinterpret_cast<float4*>(buf + kAmp);
#pragma unroll
    for (int i = 0; i < kMaxHist; ++i) {
      int c = lane + 32 * i;
      if (c < nvec) dst[c] = regs[i];
    }
  }
  // ---- current observation -------------------------------------------------------------------
  store_amp_obs_sim(buf, lane, a, e);
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_amp_obs(const pulse_amp_obs_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_amp_obs: null args");
  PULSE_REQUIRE(num_envs >= 0, "pulse_amp_obs: negative num_envs");
  if (num_envs == 0) return PULSE_OK;
  const pulse_amp_obs_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.dof_pos && a.dof_vel && a.amp_obs_buf, "pulse_amp_obs: null buffer");
  PULSE_REQUIRE(a.num_steps >= 1 && a.num_steps <= 16, "pulse_amp_obs: num_steps %d outside [1,16]", a.num_steps);
  PULSE_REQUIRE(aligned16(a.amp_obs_buf), "pulse_amp_obs: amp_obs_buf not 16-byte aligned");
  PULSE_REQUIRE(a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "pulse_amp_obs: body_env_stride too small");
  const long long threads = num_envs * 32;
  amp_obs_kernel<<<static_cast<unsigned>((threads + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("amp_obs_kernel");
  return PULSE_OK;
}
