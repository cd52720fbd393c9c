// Reference-state reset of the latent-space tasks (reach, speed, strike) on the device, no host synchronisation.  Three launches:
//   reset_compact_kernel  (reset_warps.cuh) one CTA: the ordered compaction of the reset mask or id list into the ascending env list,
//                         the humanoid and target actor lists and a device-side count;
//   ztask_reset_kernel    one warp per (reset env, AMP history step k): the shared reset_warps work (clip, start time, MotionLib
//                         gather, SMPL ground fix, _set_env_state, counters, AMP rows) with the task's pose adjustment and the strike
//                         target;
//   ztask_task_kernel     (pulse_ztask_reset_task) the reach / speed _reset_task over the same list, after the observation.
// pulse_reset_ztask_smplx runs the first two for the SMPL-X speed task: ztask_reset_kernel<SmplxLayout>, with the 465- / 466-float AMP
// rows and without a strike target; pulse_reset_smplx_target runs the same kernel for the SMPL-X reach and strike tasks (root xy zeroed,
// the strike target placed around it).
// The entry points, argument structs and Philox word layout are documented in include/pulse_b200.h.
#include "reset_warps.cuh"

namespace pulse {
namespace {

constexpr unsigned long long kStrikeStream = 1ull << 32;   // Philox index e + 2^32: strike bearing / yaw
constexpr unsigned long long kTaskStream = 2ull << 32;     // Philox index e + 2^33: _reset_task draws

template <class L, class Lib>
__global__ void __launch_bounds__(kResetWarps * 32) ztask_reset_kernel(const Lib lib, const pulse_ztask_reset_args_t a) {
  __shared__ float stage_all[kResetWarps][L::kAmpObs];
  const bool upright = a.upright != 0;
  const auto adjust = [&](long long e, int lane, const Philox4& r0, unsigned long long off, Vec3& p, Quat& rq, Vec3& v, Vec3& rp, Quat& rr,
                          Vec3& rv, Vec3& rw) {
    if (a.pose_mode == PULSE_ZPOSE_FACE_X) {   // humanoid_speed.py:251-270
      float hs, hc;
      heading_half(base_rot_removed(rr, upright), hs, hc);
      const Quat h_inv = {0.0f, 0.0f, -hs, hc};
      p = qrot(h_inv, p - rp) + rp;
      rq = qmul(h_inv, rq);
      v = qrot(h_inv, v);
      rr = qmul(h_inv, rr);
      rv = qrot(h_inv, rv);
      rw = qrot(h_inv, rw);
    } else if (a.pose_mode == PULSE_ZPOSE_ROOT_XY_ZERO) {   // humanoid_reach.py:46-48, humanoid_strike.py:147-150: the root only
      rp.x = 0.0f;
      rp.y = 0.0f;
    }
    if (lane == 0 && a.target_states != nullptr) {   // _reset_target (humanoid_strike.py:124-145), around the new root
      Philox4 r1{0u, 0u, 0u, 0u};
      if (a.strike_u == nullptr) r1 = philox4x32_10(a.seed, static_cast<unsigned long long>(e) + kStrikeStream, off);
      const float* su = a.strike_u != nullptr ? a.strike_u + 4 * e : nullptr;
      const float u_near = su ? su[0] : u01(r0.z), u_dist = su ? su[1] : u01(r0.w);
      const float u_bear = su ? su[2] : u01(r1.x), u_yaw = su ? su[3] : u01(r1.y);
      const float two_pi = static_cast<float>(2.0 * 3.14159265358979323846);
      const float dist_max = u_near < a.near_prob ? a.near_dist : a.tar_dist_max;
      const float dist = __fadd_rn(__fmul_rn(__fsub_rn(dist_max, a.tar_dist_min), u_dist), a.tar_dist_min);
      const float theta = __fmul_rn(two_pi, u_bear), yaw = __fmul_rn(two_pi, u_yaw);
      float* ts = a.target_states + e * a.target_env_stride;
      ts[0] = __fadd_rn(__fmul_rn(dist, cosf(theta)), rp.x);
      ts[1] = __fadd_rn(__fmul_rn(dist, sinf(theta)), rp.y);
      ts[2] = 0.9f;
      ts[3] = 0.0f; ts[4] = 0.0f; ts[5] = sinf(0.5f * yaw); ts[6] = cosf(0.5f * yaw);
      for (int c = 7; c < 13; ++c) ts[c] = 0.0f;
    }
  };
  reset_warps<L>(lib, a, a.target_states != nullptr && a.strike_u == nullptr, stage_all[threadIdx.x >> 5], adjust);
}

__global__ void __launch_bounds__(256) ztask_task_kernel(const pulse_ztask_task_args_t a) {
  const long long n = *a.count;
  const unsigned long long off = a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull);
  const unsigned long long span = static_cast<unsigned long long>(a.steps_max - a.steps_min);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = a.env_list[i];
    Philox4 r{0u, 0u, 0u, 0u};
    if (a.rand == nullptr || a.steps_in == nullptr) r = philox4x32_10(a.seed, static_cast<unsigned long long>(e) + kTaskStream, off);
    const long long steps = a.steps_in != nullptr ? a.steps_in[e] : a.steps_min + static_cast<long long>((static_cast<unsigned long long>(r.w) * span) >> 32);
    if (a.kind == PULSE_ZTASK_REACH) {   // humanoid_reach.py:134-146
      const float u0 = a.rand ? a.rand[3 * e] : u01(r.x), u1 = a.rand ? a.rand[3 * e + 1] : u01(r.y), u2 = a.rand ? a.rand[3 * e + 2] : u01(r.z);
      a.tar_pos[3 * e + 0] = __fmul_rn(a.dist_max, __fsub_rn(__fmul_rn(2.0f, u0), 1.0f));
      a.tar_pos[3 * e + 1] = __fmul_rn(a.dist_max, __fsub_rn(__fmul_rn(2.0f, u1), 1.0f));
      a.tar_pos[3 * e + 2] = __fadd_rn(__fmul_rn(a.height_scale, u2), a.height_min);
    } else {                             // humanoid_speed.py:166-175
      const float u = a.rand ? a.rand[e] : u01(r.x);
      a.tar_speed[e] = __fadd_rn(__fmul_rn(a.speed_scale, u), a.speed_min);
    }
    a.change_steps[e] = a.progress_buf[e] + steps;
  }
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_reset_ztask(const pulse_motionlib_t* lib, const pulse_ztask_reset_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "pulse_reset_ztask: null lib/args");
  const pulse_ztask_reset_args_t& a = *args;
  PULSE_REQUIRE(num_envs >= 0 && num_envs < (1ll << 31), "pulse_reset_ztask: num_envs %lld outside [0, 2^31)", (long long)num_envs);
  PULSE_REQUIRE(a.reset_buf != nullptr || a.env_ids_in != nullptr, "pulse_reset_ztask: neither a reset mask nor an env id list");
  PULSE_REQUIRE(a.env_ids_in == nullptr || (a.num_ids >= 0 && a.num_ids <= num_envs), "pulse_reset_ztask: num_ids %lld outside [0, %lld]",
                (long long)a.num_ids, (long long)num_envs);
  PULSE_REQUIRE(a.env_list != nullptr && a.count != nullptr, "pulse_reset_ztask: env_list / count outputs are required");
  PULSE_REQUIRE(a.sampled_motion_ids && a.motion_start_times && a.progress_buf, "pulse_reset_ztask: null task buffer");
  PULSE_REQUIRE(a.root_states && a.dof_pos && a.dof_vel && a.rigid_body_state, "pulse_reset_ztask: null simulator tensor");
  PULSE_REQUIRE(a.root_env_stride >= PULSE_BODY_STATE_W && a.dof_elem_stride >= 1 && a.dof_env_stride >= PULSE_NUM_DOF * a.dof_elem_stride &&
                a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "pulse_reset_ztask: bad root / dof / rigid-body strides");
  PULSE_REQUIRE(a.contact_forces == nullptr || (a.contact_bodies >= 0 && a.contact_env_stride >= 3 * a.contact_bodies),
                "pulse_reset_ztask: bad contact-force strides");
  PULSE_REQUIRE(a.target_states == nullptr || a.target_env_stride >= PULSE_BODY_STATE_W, "pulse_reset_ztask: bad target_states stride");
  PULSE_REQUIRE(a.floor != nullptr && a.floor_len >= lib->d.total_frames, "pulse_reset_ztask: floor table of %lld frames, the MotionLib has %lld",
                (long long)a.floor_len, (long long)lib->d.total_frames);
  PULSE_REQUIRE(a.motion_ids_in != nullptr || (a.sampling_cdf != nullptr && lib->d.num_motions >= 1),
                "pulse_reset_ztask: null sampling_cdf (needed to draw the clips)");
  PULSE_REQUIRE(a.pose_mode >= PULSE_ZPOSE_AS_IS && a.pose_mode <= PULSE_ZPOSE_FACE_X, "pulse_reset_ztask: unknown pose_mode %d", a.pose_mode);
  PULSE_REQUIRE(a.state_init == PULSE_ZINIT_RANDOM || a.state_init == PULSE_ZINIT_START, "pulse_reset_ztask: unknown state_init %d", a.state_init);
  PULSE_REQUIRE(a.amp_obs_buf == nullptr || (a.num_amp_steps >= 1 && a.num_amp_steps <= 16), "pulse_reset_ztask: num_amp_steps outside [1,16]");
  PULSE_REQUIRE(a.amp_fresh == nullptr || a.amp_obs_buf != nullptr, "pulse_reset_ztask: amp_fresh flags need the back-filled amp_obs_buf");
  PULSE_REQUIRE(a.amp_obs_buf == nullptr || a.amp_width == PULSE_AMP_OBS || a.amp_width == PULSE_AMP_OBS_NO_HEIGHT,
                "pulse_reset_ztask: amp_width %d is neither %d nor %d", a.amp_width, PULSE_AMP_OBS, PULSE_AMP_OBS_NO_HEIGHT);
  PULSE_REQUIRE(lib->d.aux_rec != nullptr, "pulse_reset_ztask: the MotionLib handle has no aux records (dof_pos / dof_vel)");
  if (num_envs == 0) return PULSE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  reset_compact_kernel<<<1, kCompactThreads, 0, st>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("reset_compact_kernel");
  const long long upper = (a.env_ids_in != nullptr ? a.num_ids : num_envs) * (a.amp_obs_buf != nullptr ? a.num_amp_steps : 1);
  ztask_reset_kernel<SmplLayout><<<grid_for(upper, kResetWarps), kResetWarps * 32, 0, st>>>(lib->d, a);
  PULSE_LAUNCH_OK("ztask_reset_kernel");
  return PULSE_OK;
}

extern "C" int pulse_ztask_reset_task(const pulse_ztask_task_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_ztask_reset_task: null args");
  const pulse_ztask_task_args_t& a = *args;
  PULSE_REQUIRE(num_envs >= 0 && num_envs < (1ll << 31), "pulse_ztask_reset_task: num_envs %lld outside [0, 2^31)", (long long)num_envs);
  PULSE_REQUIRE(a.kind == PULSE_ZTASK_REACH || a.kind == PULSE_ZTASK_SPEED, "pulse_ztask_reset_task: unknown task kind %d", a.kind);
  PULSE_REQUIRE(a.env_list && a.count && a.progress_buf && a.change_steps, "pulse_ztask_reset_task: null list / count / task buffer");
  PULSE_REQUIRE(a.kind != PULSE_ZTASK_REACH || a.tar_pos != nullptr, "pulse_ztask_reset_task: the reach task needs tar_pos");
  PULSE_REQUIRE(a.kind != PULSE_ZTASK_SPEED || a.tar_speed != nullptr, "pulse_ztask_reset_task: the speed task needs tar_speed");
  PULSE_REQUIRE(a.steps_in != nullptr || a.steps_max > a.steps_min, "pulse_ztask_reset_task: empty randint range [%lld, %lld)",
                (long long)a.steps_min, (long long)a.steps_max);
  if (num_envs == 0) return PULSE_OK;
  ztask_task_kernel<<<grid_for(num_envs, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  PULSE_LAUNCH_OK("ztask_task_kernel");
  return PULSE_OK;
}

namespace pulse {
namespace {
// The checks pulse_reset_ztask_smplx and pulse_reset_smplx_target share (`who` prefixes the messages), then their two launches.
int reset_smplx(const pulse_smplx_motionlib_t* lib, const pulse_ztask_reset_args_t* args, int64_t num_envs, void* stream, const char* who) {
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "%s: null lib/args", who);
  const pulse_ztask_reset_args_t& a = *args;
  PULSE_REQUIRE(num_envs >= 0 && num_envs < (1ll << 31), "%s: num_envs %lld outside [0, 2^31)", who, (long long)num_envs);
  PULSE_REQUIRE(a.reset_buf != nullptr || a.env_ids_in != nullptr, "%s: neither a reset mask nor an env id list", who);
  PULSE_REQUIRE(a.env_ids_in == nullptr || (a.num_ids >= 0 && a.num_ids <= num_envs), "%s: num_ids %lld outside [0, %lld]", who,
                (long long)a.num_ids, (long long)num_envs);
  PULSE_REQUIRE(a.env_list != nullptr && a.count != nullptr, "%s: env_list / count outputs are required", who);
  PULSE_REQUIRE(a.sampled_motion_ids && a.motion_start_times && a.progress_buf, "%s: null task buffer", who);
  PULSE_REQUIRE(a.root_states && a.dof_pos && a.dof_vel && a.rigid_body_state, "%s: null simulator tensor", who);
  PULSE_REQUIRE(a.root_env_stride >= PULSE_BODY_STATE_W && a.dof_elem_stride >= 1 && a.dof_env_stride >= PULSE_SMPLX_DOF * a.dof_elem_stride &&
                a.body_env_stride >= PULSE_SMPLX_BODIES * PULSE_BODY_STATE_W, "%s: bad root / dof / rigid-body strides", who);
  PULSE_REQUIRE(a.contact_forces == nullptr || (a.contact_bodies >= 0 && a.contact_env_stride >= 3 * a.contact_bodies),
                "%s: bad contact-force strides", who);
  PULSE_REQUIRE(a.amp_obs_buf == nullptr || (a.num_amp_steps >= 1 && a.num_amp_steps <= 16),
                "%s: the AMP history back-fill takes num_amp_steps in [1,16], not %d", who, a.num_amp_steps);
  PULSE_REQUIRE(a.amp_obs_buf == nullptr || a.amp_width == PULSE_SMPLX_AMP_OBS || a.amp_width == PULSE_SMPLX_AMP_OBS_NO_HEIGHT,
                "%s: AMP amp_width %d is neither %d nor %d (the SMPL-X rows)", who, a.amp_width, PULSE_SMPLX_AMP_OBS,
                PULSE_SMPLX_AMP_OBS_NO_HEIGHT);
  PULSE_REQUIRE(a.amp_fresh == nullptr || a.amp_obs_buf != nullptr, "%s: amp_fresh flags need the back-filled AMP amp_obs_buf", who);
  PULSE_REQUIRE(a.floor != nullptr && a.floor_len >= lib->d.total_frames, "%s: floor table of %lld frames, the MotionLib has %lld", who,
                (long long)a.floor_len, (long long)lib->d.total_frames);
  PULSE_REQUIRE(a.motion_ids_in != nullptr || a.sampling_cdf != nullptr, "%s: null sampling_cdf (needed to draw the clips)", who);
  PULSE_REQUIRE(a.state_init == PULSE_ZINIT_RANDOM || a.state_init == PULSE_ZINIT_START, "%s: unknown state_init %d", who, a.state_init);
  if (num_envs == 0) return PULSE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  reset_compact_kernel<<<1, kCompactThreads, 0, st>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("reset_compact_kernel");
  const long long upper = (a.env_ids_in != nullptr ? a.num_ids : num_envs) * (a.amp_obs_buf != nullptr ? a.num_amp_steps : 1);
  ztask_reset_kernel<SmplxLayout><<<grid_for(upper, kResetWarps), kResetWarps * 32, 0, st>>>(lib->d, a);
  PULSE_LAUNCH_OK("ztask_reset_kernel<SmplxLayout>");
  return PULSE_OK;
}
}  // namespace
}  // namespace pulse

extern "C" int pulse_reset_ztask_smplx(const pulse_smplx_motionlib_t* lib, const pulse_ztask_reset_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_reset_ztask_smplx: null lib/args");
  PULSE_REQUIRE(args->target_states == nullptr, "pulse_reset_ztask_smplx: the SMPL-X reset serves the speed task (target_states must be NULL)");
  PULSE_REQUIRE(args->pose_mode == PULSE_ZPOSE_FACE_X, "pulse_reset_ztask_smplx: pose_mode %d, the speed task's is PULSE_ZPOSE_FACE_X",
                args->pose_mode);
  return reset_smplx(lib, args, num_envs, stream, "pulse_reset_ztask_smplx");
}

extern "C" int pulse_reset_smplx_target(const pulse_smplx_motionlib_t* lib, const pulse_ztask_reset_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_reset_smplx_target: null lib/args");
  PULSE_REQUIRE(args->pose_mode == PULSE_ZPOSE_ROOT_XY_ZERO, "pulse_reset_smplx_target: pose_mode %d, the reach and strike tasks' is "
                "PULSE_ZPOSE_ROOT_XY_ZERO", args->pose_mode);
  PULSE_REQUIRE(args->target_states == nullptr || args->target_env_stride >= PULSE_BODY_STATE_W,
                "pulse_reset_smplx_target: bad target_states stride");
  return reset_smplx(lib, args, num_envs, stream, "pulse_reset_smplx_target");
}
