// Rollout glue of AMPAgent.play_steps (phc/learning/amp_agent.py:341-439) as three row-wise kernels that write STRAIGHT into the
// experience-buffer slices (pointer + stride), so the per-step ATen copies / elementwise chains of round 1 disappear:
//   policy_post_kernel  ModelA2CContinuousLogStd sampling [rl_games]: a = mu + sigma * eps with eps drawn in-kernel (Philox4x32-10 or
//                       injected), neglogp, value de-normalisation (RunningMeanStd.forward(unnorm=True), running_mean_std.py:84-87),
//                       PD targets (Humanoid._action_to_pd_targets, humanoid.py:1392-1394) -- get_action_values + the experience
//                       buffer updates of amp_agent.py:361-378 + pre_physics_step's target computation in ONE launch;
//   value_post_kernel   next_values = unnormalise(critic(next obs)) * (1 - terminated)  (amp_agent.py:396-398);
//   amp_row_kernel      this step's AMP observation row [cur | previous row's first (steps-1)*196 floats] written directly into the
//                       experience slice (humanoid_amp.py:622-667 + amp_agent.py:385): 7 056 B read + 7 840 B written per env instead
//                       of the in-place shift (7 056 + 7 840) followed by a 7 840 + 7 840 B copy.  Envs reset since the last step take
//                       their previous row from the rows `pulse_reset_ref_state` back-filled (`fresh` flags, cleared here).
//   amp_row_any_kernel  the same row in the other layouts the resets write: 195 floats (no root height; rows are 780 B, so not
//                       16-byte units) and / or the remove_base_rot heading of a non-upright start; instantiated for SMPL-X
//                       (pulse_smplx_amp_obs_row, 466 / 465 floats, not 16-byte units either).
#include "philox.cuh"
#include "motion_amp.cuh"
#include "value_unnorm.cuh"

namespace pulse {
namespace {

__global__ void __launch_bounds__(128) policy_post_kernel(const pulse_policy_post_args_t a, long long rows) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int A = a.num_actions;
  const unsigned long long off = a.rng_offset != nullptr ? *a.rng_offset + a.rng_step : a.rng_step;
  // Philox indices per row: 64 (pairs p < 64) up to 128 actions, 128 above, so no two rows share a block (pulse_b200.h)
  const unsigned long long row_blocks = A <= 128 ? 64ull : 128ull;
  float acc = 0.0f, ls = 0.0f;
  // lanes take PAIRS of actions (2*lane + 64*i): one Philox call yields four words = two Box-Muller pairs
  for (int i = 0; 2 * lane + 64 * i < A; ++i) {
    const int k0 = 2 * lane + 64 * i;
    float e0, e1;
    if (a.eps != nullptr) {
      e0 = a.eps[row * a.ld_eps + k0];
      e1 = k0 + 1 < A ? a.eps[row * a.ld_eps + k0 + 1] : 0.0f;
    } else {
      const Philox4 r = philox4x32_10(a.seed, static_cast<unsigned long long>(row) * row_blocks + static_cast<unsigned long long>(lane + 32 * i), off);
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
      if (a.mus_out != nullptr) a.mus_out[row * a.ld_mus + k] = m;
      if (a.pd_targets != nullptr) {
        const float tgt = __fadd_rn(a.pd_offset[k], __fmul_rn(a.pd_scale[k], act));     // humanoid.py:1392-1394
        a.pd_targets[row * a.ld_pd + k] = tgt;
      }
      const float z = (act - m) / sg;
      acc += z * z;
      ls += l;
    }
  }
  acc = warp_sum(acc);
  ls = warp_sum(ls);
  if (lane == 0) {
    a.neglogp[row * a.ld_neglogp] = 0.5f * acc + 0.5f * 1.8378770664093453f * A + ls;   // log(2*pi)
    if (a.values_out != nullptr) a.values_out[row * a.ld_values] = value_unnorm(a.value[row * a.ld_value], a.value_mean, a.value_var, a.value_eps);
  }
}

__global__ void __launch_bounds__(256) value_post_kernel(const float* __restrict__ value, long long ld_value, const double* mean, const double* var,
                                                         float eps, const long long* __restrict__ terminate, float* __restrict__ out,
                                                         long long ld_out, long long rows) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float v = value_unnorm(value[r * ld_value], mean, var, eps);
  if (terminate != nullptr) v = __fmul_rn(v, __fsub_rn(1.0f, static_cast<float>(terminate[r])));   // next_vals *= (1.0 - terminated)
  out[r * ld_out] = v;
}

constexpr int kAmp = PULSE_AMP_OBS;

__global__ void __launch_bounds__(128) amp_row_kernel(const pulse_amp_row_args_t a, long long n) {
  const long long e = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= n) return;
  float* out = a.out + e * a.ld_out;
  const int hist = (a.num_steps - 1) * kAmp;
  // ---- history part: out[196 + k] <- prev[k], k < hist (prev and out never alias: different experience slices) ------------------
  const bool fresh = a.fresh != nullptr && a.fresh[e] != 0;
  const float* prev = fresh ? a.fresh_rows + e * (long long)a.num_steps * kAmp : a.prev + e * a.ld_prev;
  {
    // (steps-1)*49 16-byte units per env (441 for 10 steps): all loads of the warp are issued before the first store (16 in flight per lane)
    const float4* src = reinterpret_cast<const float4*>(prev);
    float4* dst = reinterpret_cast<float4*>(out + kAmp);
    const int nvec = hist / 4;
    float4 regs[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) regs[i] = __ldcs(src + c);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) __stcs(dst + c, regs[i]);
    }
    for (int c = lane + 512; c < nvec; c += 32) dst[c] = src[c];   // more than 11 history steps
  }
  __syncwarp();   // every lane has read the flag before lane 0 clears it
  if (fresh && lane == 0) a.fresh[e] = 0;
  // ---- current observation -------------------------------------------------------------------------------------------------------
  store_amp_obs_sim(out, lane, a, e);
}

constexpr int kAmpRowWarps = 4;

template <class L>
__global__ void __launch_bounds__(kAmpRowWarps * 32) amp_row_any_kernel(const pulse_amp_row_args_t a, int width, long long n) {
  __shared__ float stage_all[kAmpRowWarps][L::kAmpObs];
  const long long e = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= n) return;
  float* out = a.out + e * a.ld_out;
  const bool fresh = a.fresh != nullptr && a.fresh[e] != 0;
  const float* prev = fresh ? a.fresh_rows + e * (long long)a.num_steps * width : a.prev + e * a.ld_prev;
  const int hist = (a.num_steps - 1) * width;
  for (int c = lane; c < hist; c += 32) __stcs(out + width + c, __ldcs(prev + c));
  __syncwarp();   // every lane has read the flag before lane 0 clears it
  if (fresh && lane == 0) a.fresh[e] = 0;
  const float* bs = a.body_state + e * a.body_env_stride;
  const float* dp = a.dof_pos + e * a.dof_env_stride;
  const float* dv = a.dof_vel + e * a.dof_env_stride;
  const long long ds = a.dof_elem_stride;
  const auto joint = [&](int jt) {
    return AmpJoint{{dp[(3 * jt + 0) * ds], dp[(3 * jt + 1) * ds], dp[(3 * jt + 2) * ds]},
                    {dv[(3 * jt + 0) * ds], dv[(3 * jt + 1) * ds], dv[(3 * jt + 2) * ds]}};
  };
  const auto key_pos = [&](int kb) { return ldv(bs + kb * PULSE_BODY_STATE_W); };
  store_amp_row<L>(out, width, stage_all[threadIdx.x >> 5], lane, ldv(bs), ldq(bs + 3), ldv(bs + 7), ldv(bs + 10), a.remove_base_rot == 0, joint,
                   key_pos);
}

__global__ void bump_counter_kernel(unsigned long long* c, unsigned long long by) { *c += by; }

}  // namespace
}  // namespace pulse

extern "C" int pulse_policy_post(const pulse_policy_post_args_t* args, int64_t rows, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_policy_post: null args");
  PULSE_REQUIRE(rows >= 0, "pulse_policy_post: negative rows");
  if (rows == 0) return PULSE_OK;
  const pulse_policy_post_args_t& a = *args;
  PULSE_REQUIRE(a.mu && a.logstd && a.actions && a.neglogp, "pulse_policy_post: null mu / logstd / actions / neglogp");
  PULSE_REQUIRE(a.num_actions >= 1 && a.num_actions <= 256, "pulse_policy_post: num_actions %d outside [1,256]", a.num_actions);
  PULSE_REQUIRE(a.ld_mu >= a.num_actions && a.ld_actions >= a.num_actions && a.ld_neglogp >= 1, "pulse_policy_post: leading dimensions too small");
  PULSE_REQUIRE(a.eps == nullptr || a.ld_eps >= a.num_actions, "pulse_policy_post: ld_eps too small");
  PULSE_REQUIRE(a.mus_out == nullptr || a.ld_mus >= a.num_actions, "pulse_policy_post: ld_mus too small");
  PULSE_REQUIRE(a.values_out == nullptr || (a.value != nullptr && a.ld_value >= 1 && a.ld_values >= 1), "pulse_policy_post: values_out needs value");
  PULSE_REQUIRE((a.value_mean == nullptr) == (a.value_var == nullptr), "pulse_policy_post: value_mean and value_var go together");
  PULSE_REQUIRE(a.pd_targets == nullptr || (a.pd_offset && a.pd_scale && a.ld_pd >= a.num_actions), "pulse_policy_post: pd_targets needs offset / scale");
  policy_post_kernel<<<static_cast<unsigned>((rows * 32 + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)rows);
  PULSE_LAUNCH_OK("policy_post_kernel");
  return PULSE_OK;
}

extern "C" int pulse_value_post(const float* value, int64_t ld_value, const double* mean, const double* var, float eps, const int64_t* terminate,
                                float* out, int64_t ld_out, int64_t rows, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(value != nullptr && out != nullptr, "pulse_value_post: null value / out");
  PULSE_REQUIRE(rows >= 0 && ld_value >= 1 && ld_out >= 1, "pulse_value_post: bad sizes");
  PULSE_REQUIRE((mean == nullptr) == (var == nullptr), "pulse_value_post: mean and var go together");
  if (rows == 0) return PULSE_OK;
  value_post_kernel<<<static_cast<unsigned>((rows + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      value, ld_value, mean, var, eps, reinterpret_cast<const long long*>(terminate), out, ld_out, (long long)rows);
  PULSE_LAUNCH_OK("value_post_kernel");
  return PULSE_OK;
}

extern "C" int pulse_amp_obs_row(const pulse_amp_row_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_amp_obs_row: null args");
  PULSE_REQUIRE(num_envs >= 0, "pulse_amp_obs_row: negative num_envs");
  if (num_envs == 0) return PULSE_OK;
  const pulse_amp_row_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.dof_pos && a.dof_vel && a.prev && a.out, "pulse_amp_obs_row: null buffer");
  PULSE_REQUIRE(a.num_steps >= 1 && a.num_steps <= 16, "pulse_amp_obs_row: num_steps %d outside [1,16]", a.num_steps);
  PULSE_REQUIRE(a.amp_width == 0 || a.amp_width == PULSE_AMP_OBS || a.amp_width == PULSE_AMP_OBS_NO_HEIGHT,
                "pulse_amp_obs_row: amp_width %d is neither %d nor %d", a.amp_width, PULSE_AMP_OBS, PULSE_AMP_OBS_NO_HEIGHT);
  const int width = a.amp_width == 0 ? PULSE_AMP_OBS : a.amp_width;
  PULSE_REQUIRE(a.ld_prev >= (a.num_steps - 1) * width && a.ld_out >= a.num_steps * width, "pulse_amp_obs_row: row strides too small");
  PULSE_REQUIRE(a.prev != a.out, "pulse_amp_obs_row: prev and out must be different experience slices (use pulse_amp_obs for the in-place shift)");
  PULSE_REQUIRE((a.fresh == nullptr) == (a.fresh_rows == nullptr), "pulse_amp_obs_row: fresh flags and fresh_rows go together");
  PULSE_REQUIRE(a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "pulse_amp_obs_row: body_env_stride too small");
  if (width != PULSE_AMP_OBS || a.remove_base_rot != 0) {
    amp_row_any_kernel<SmplLayout><<<static_cast<unsigned>((num_envs + kAmpRowWarps - 1) / kAmpRowWarps), kAmpRowWarps * 32, 0,
                                     static_cast<cudaStream_t>(stream)>>>(a, width, (long long)num_envs);
    PULSE_LAUNCH_OK("amp_row_any_kernel");
    return PULSE_OK;
  }
  PULSE_REQUIRE(aligned16(a.prev) && aligned16(a.out) && (a.ld_prev % 4) == 0 && (a.ld_out % 4) == 0, "pulse_amp_obs_row: rows must be 16-byte aligned");
  PULSE_REQUIRE(a.fresh_rows == nullptr || aligned16(a.fresh_rows), "pulse_amp_obs_row: fresh_rows not 16-byte aligned");
  const long long threads = num_envs * 32;
  amp_row_kernel<<<static_cast<unsigned>((threads + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("amp_row_kernel");
  return PULSE_OK;
}

extern "C" int pulse_smplx_amp_obs_row(const pulse_amp_row_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_smplx_amp_obs_row: null args");
  PULSE_REQUIRE(num_envs >= 0, "pulse_smplx_amp_obs_row: negative num_envs");
  if (num_envs == 0) return PULSE_OK;
  const pulse_amp_row_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.dof_pos && a.dof_vel && a.prev && a.out, "pulse_smplx_amp_obs_row: null buffer");
  PULSE_REQUIRE(a.num_steps >= 1 && a.num_steps <= 16, "pulse_smplx_amp_obs_row: num_steps %d outside [1,16]", a.num_steps);
  PULSE_REQUIRE(a.amp_width == PULSE_SMPLX_AMP_OBS || a.amp_width == PULSE_SMPLX_AMP_OBS_NO_HEIGHT,
                "pulse_smplx_amp_obs_row: amp_width %d is neither %d nor %d", a.amp_width, PULSE_SMPLX_AMP_OBS, PULSE_SMPLX_AMP_OBS_NO_HEIGHT);
  PULSE_REQUIRE(a.remove_base_rot == 1, "pulse_smplx_amp_obs_row: the SMPL-X rows take the heading of remove_base_rot(q0) (remove_base_rot 1)");
  const int width = a.amp_width;
  PULSE_REQUIRE(a.ld_prev >= (a.num_steps - 1) * width && a.ld_out >= a.num_steps * width, "pulse_smplx_amp_obs_row: row strides too small");
  PULSE_REQUIRE(a.prev != a.out, "pulse_smplx_amp_obs_row: prev and out must be different experience slices");
  PULSE_REQUIRE((a.fresh == nullptr) == (a.fresh_rows == nullptr), "pulse_smplx_amp_obs_row: fresh flags and fresh_rows go together");
  PULSE_REQUIRE(a.body_env_stride >= PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W, "pulse_smplx_amp_obs_row: body_env_stride too small");
  PULSE_REQUIRE(a.dof_elem_stride >= 1 && a.dof_env_stride >= PULSE_SMPLX_DOF * a.dof_elem_stride, "pulse_smplx_amp_obs_row: dof strides too small");
  amp_row_any_kernel<SmplxLayout><<<static_cast<unsigned>((num_envs + kAmpRowWarps - 1) / kAmpRowWarps), kAmpRowWarps * 32, 0,
                                    static_cast<cudaStream_t>(stream)>>>(a, width, (long long)num_envs);
  PULSE_LAUNCH_OK("amp_row_any_kernel<SmplxLayout>");
  return PULSE_OK;
}

extern "C" int pulse_bump_counter(uint64_t* counter, uint64_t by, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(counter != nullptr, "pulse_bump_counter: null counter");
  bump_counter_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<unsigned long long*>(counter), by);
  PULSE_LAUNCH_OK("bump_counter_kernel");
  return PULSE_OK;
}

// ---- timing events that survive CUDA-graph capture ---------------------------------------------------------------------------
// torch.cuda.Event.record() inside a capture becomes an internal dependency node that cannot be queried; bench.py has to time the
// fused step kernel LIVE inside the timed region even when the whole rollout is one graph, so these wrap cudaEventRecordWithFlags
// (cudaEventRecordExternal): captured as an event-record NODE, the event is re-recorded by every replay and elapsed times can be read.
extern "C" int pulse_event_create(void** event) {
  using namespace pulse;
  PULSE_REQUIRE(event != nullptr, "pulse_event_create: null out pointer");
  cudaEvent_t e;
  PULSE_CUDA_OK(cudaEventCreate(&e));
  *event = e;
  return PULSE_OK;
}
extern "C" int pulse_event_destroy(void* event) {
  using namespace pulse;
  if (event != nullptr) PULSE_CUDA_OK(cudaEventDestroy(static_cast<cudaEvent_t>(event)));
  return PULSE_OK;
}
extern "C" int pulse_event_record(void* event, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(event != nullptr, "pulse_event_record: null event");
  // the external flag is only legal while the stream is being captured; outside a capture this is an ordinary record
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  PULSE_CUDA_OK(cudaStreamIsCapturing(static_cast<cudaStream_t>(stream), &st));
  PULSE_CUDA_OK(cudaEventRecordWithFlags(static_cast<cudaEvent_t>(event), static_cast<cudaStream_t>(stream),
                                         st == cudaStreamCaptureStatusActive ? cudaEventRecordExternal : cudaEventRecordDefault));
  return PULSE_OK;
}
extern "C" int pulse_event_elapsed_ms(void* start, void* stop, float* ms) {
  using namespace pulse;
  PULSE_REQUIRE(start != nullptr && stop != nullptr && ms != nullptr, "pulse_event_elapsed_ms: null argument");
  PULSE_CUDA_OK(cudaEventElapsedTime(ms, static_cast<cudaEvent_t>(start), static_cast<cudaEvent_t>(stop)));
  return PULSE_OK;
}
