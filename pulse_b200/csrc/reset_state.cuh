// Device code of the reference-state reset, shared by pulse_reset_ref_state (reset.cu) and pulse_reset_getup (getup_reset.cu):
//   compact_slot            one round of the ordered block-wide compaction (ballot / prefix scan, no atomics: the order is
//                           deterministic) that turns a reset mask or an id list into an ascending env list;
//   reset_ref_state_kernel  one warp per (reset env, AMP history step k): start time = sample_time_interval
//                           (motion_lib_base.py:411-420), MotionLib query at t0 - k*dt (get_motion_state :434-517); k = 0 scatters the
//                           reference pose into the simulator's root / dof / rigid-body views (_set_env_state, humanoid_amp.py:565-597)
//                           and clears the task counters (_reset_ref_state_init humanoid_im.py:921-948, _reset_env_tensors
//                           humanoid.py:589-609); every k writes its AMP observation row (_init_amp_obs, humanoid_amp.py:519-563).
// HBM-bound gather / scatter: ~44 KB of packed frame records per reset env (20 rows x 2 208 B), ~11 KB written.
#pragma once
#include "compact.cuh"
#include "philox.cuh"
#include "humanoid_obs.cuh"

namespace pulse {
namespace {

// Env behind candidate i of a reset set: entry i of the explicit id list, or i itself when reset_buf[i] != 0 (mask mode); -1 if none.
__device__ __forceinline__ long long reset_candidate(const pulse_reset_args_t& a, long long i, long long n) {
  if (i >= n) return -1;
  if (a.env_ids_in != nullptr) return a.env_ids_in[i];
  return a.reset_buf[i] != 0 ? i : -1;
}

__global__ void __launch_bounds__(256) reset_ref_state_kernel(const pulse_motionlib_desc_t lib, const pulse_reset_args_t a) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int steps = a.amp_obs_buf != nullptr ? a.num_amp_steps : 1;
  const long long items = static_cast<long long>(*a.count) * steps;
  const float step30 = static_cast<float>(1.0 / 30.0);   // `curr_fps = 1 / 30` (python double) meets fp32 tensors as fp32(1/30)
  for (long long it = warp0; it < items; it += nwarps) {
    const long long i = it / steps;
    const int k = static_cast<int>(it - i * steps);
    const long long e = a.env_list[i];
    const long long mid = a.motion_ids[e];
    const float mlen = lib.lengths[mid];
    float ph;
    if (a.phase != nullptr) ph = a.phase[e];
    else ph = philox_uniform(a.seed, static_cast<unsigned long long>(e), a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull));
    // ((phase * motion_len) / curr_fps).long() * curr_fps
    const float t0 = __fmul_rn(__ll2float_rn(static_cast<long long>(__fdiv_rn(__fmul_rn(ph, mlen), step30))), step30);
    // _init_amp_obs_ref: motion_times + (-dt * (arange + 1)) (humanoid_amp.py:540-542); k = 0 is the reset pose itself
    const float t = k == 0 ? t0 : __fadd_rn(t0, __fmul_rn(-a.dt, static_cast<float>(k)));
    long long i0, i1;
    float b;
    frame_blend_rn(t, mlen, lib.num_frames[mid], lib.dt[mid], i0, i1, b);
    const long long f0 = i0 + lib.length_starts[mid], f1 = i1 + lib.length_starts[mid];
    const float* r0 = lib.frame_rec + f0 * PULSE_FRAME_REC;
    const float* r1 = lib.frame_rec + f1 * PULSE_FRAME_REC;
    const float* x0 = lib.aux_rec + f0 * PULSE_AUX_REC;
    const float* x1 = lib.aux_rec + f1 * PULSE_AUX_REC;
    // root state of the query (every lane: broadcast loads): the frame of the AMP features
    Vec3 p0, v0, w0;
    p0.x = lerp_rn(r0[0], r1[0], b); p0.y = lerp_rn(r0[1], r1[1], b); p0.z = lerp_rn(r0[2], r1[2], b);
    v0.x = lerp_rn(r0[168], r1[168], b); v0.y = lerp_rn(r0[169], r1[169], b); v0.z = lerp_rn(r0[170], r1[170], b);
    w0.x = lerp_rn(r0[240], r1[240], b); w0.y = lerp_rn(r0[241], r1[241], b); w0.z = lerp_rn(r0[242], r1[242], b);
    const Quat q0 = slerp(ldq4(r0 + 72), ldq4(r1 + 72), b);

    if (k == 0) {
      // ---- _set_env_state: the whole reference pose into the simulator's views (global offset is 0 after the reset) --------------
      if (lane < PULSE_NUM_BODIES) {
        const int j = lane;
        Vec3 p, v, w;
        p.x = __fadd_rn(lerp_rn(r0[3 * j], r1[3 * j], b), 0.0f);
        p.y = __fadd_rn(lerp_rn(r0[3 * j + 1], r1[3 * j + 1], b), 0.0f);
        p.z = __fadd_rn(lerp_rn(r0[3 * j + 2], r1[3 * j + 2], b), 0.0f);
        v.x = lerp_rn(r0[168 + 3 * j], r1[168 + 3 * j], b);
        v.y = lerp_rn(r0[169 + 3 * j], r1[169 + 3 * j], b);
        v.z = lerp_rn(r0[170 + 3 * j], r1[170 + 3 * j], b);
        w.x = lerp_rn(r0[240 + 3 * j], r1[240 + 3 * j], b);
        w.y = lerp_rn(r0[241 + 3 * j], r1[241 + 3 * j], b);
        w.z = lerp_rn(r0[242 + 3 * j], r1[242 + 3 * j], b);
        const Quat rq = slerp(ldq4(r0 + 72 + 4 * j), ldq4(r1 + 72 + 4 * j), b);
        if (a.rigid_body_state != nullptr) {
          float* d = a.rigid_body_state + e * a.body_env_stride + j * PULSE_BODY_STATE_W;
          d[0] = p.x; d[1] = p.y; d[2] = p.z; d[3] = rq.x; d[4] = rq.y; d[5] = rq.z; d[6] = rq.w;
          d[7] = v.x; d[8] = v.y; d[9] = v.z; d[10] = w.x; d[11] = w.y; d[12] = w.z;
        }
        if (j == 0) {
          float* d = a.root_states + e * a.root_env_stride;
          d[0] = p.x; d[1] = p.y; d[2] = p.z; d[3] = rq.x; d[4] = rq.y; d[5] = rq.z; d[6] = rq.w;
          d[7] = v.x; d[8] = v.y; d[9] = v.z; d[10] = w.x; d[11] = w.y; d[12] = w.z;
        }
        if (j >= 1) {   // dof_pos = exp_map(slerp(local rotations)) of joints 1..23 (motion_lib_base.py:489-490, :561-564)
          const Vec3 em = quat_exp_map(slerp(ldq4(x0 + 4 * j), ldq4(x1 + 4 * j), b));
          float* d = a.dof_pos + e * a.dof_env_stride + 3 * (j - 1) * a.dof_elem_stride;
          d[0] = em.x; d[a.dof_elem_stride] = em.y; d[2 * a.dof_elem_stride] = em.z;
        }
      }
      for (int c = lane; c < PULSE_NUM_DOF; c += 32) a.dof_vel[e * a.dof_env_stride + c * a.dof_elem_stride] = lerp_rn(x0[96 + c], x1[96 + c], b);
      if (a.contact_forces != nullptr)
        for (int c = lane; c < a.contact_bodies * 3; c += 32) a.contact_forces[e * a.contact_env_stride + c] = 0.0f;
      if (lane == 0) {   // _reset_ref_state_init (humanoid_im.py:921-927, humanoid_amp.py:483-485) + _reset_env_tensors (humanoid.py:603-606)
        a.motion_start_times[e] = t0;
        a.motion_start_offset[e] = 0.0f;
        a.global_offset[3 * e] = 0.0f; a.global_offset[3 * e + 1] = 0.0f; a.global_offset[3 * e + 2] = 0.0f;
        if (a.cycle_counter != nullptr) a.cycle_counter[e] = 0;
        a.progress_buf[e] = 0;
        if (a.reset_buf != nullptr) a.reset_buf[e] = 0;
        if (a.terminate_buf != nullptr) a.terminate_buf[e] = 0;
        if (a.amp_fresh != nullptr) a.amp_fresh[e] = 1;
      }
    }
    if (a.amp_obs_buf == nullptr) continue;
    // ---- AMP observation of the reference motion at t (build_amp_observations_smpl, humanoid_amp.py:924-969) --------------------------
    // joint jt = body jt + 1: dof_pos = exp_map(slerp(local rotations)), dof_vel blended
    const auto joint = [&](int jt) {
      return AmpJoint{quat_exp_map(slerp(ldq4(x0 + 4 * (jt + 1)), ldq4(x1 + 4 * (jt + 1)), b)),
                      {lerp_rn(x0[96 + 3 * jt], x1[96 + 3 * jt], b), lerp_rn(x0[97 + 3 * jt], x1[97 + 3 * jt], b),
                       lerp_rn(x0[98 + 3 * jt], x1[98 + 3 * jt], b)}};
    };
    const auto key_pos = [&](int kb) {
      return Vec3{lerp_rn(r0[3 * kb], r1[3 * kb], b), lerp_rn(r0[3 * kb + 1], r1[3 * kb + 1], b), lerp_rn(r0[3 * kb + 2], r1[3 * kb + 2], b)};
    };
    store_amp_obs(a.amp_obs_buf + (e * a.num_amp_steps + k) * PULSE_AMP_OBS, lane, p0, q0, v0, w0, joint, key_pos);
  }
}

}  // namespace

// Argument checks of the reference-state part, shared by both entry points (`who` prefixes the messages).
inline int check_ref_state_args(const pulse_motionlib_t* lib, const pulse_reset_args_t& a, int64_t num_envs, const char* who) {
  PULSE_REQUIRE(num_envs >= 0, "%s: negative num_envs", who);
  PULSE_REQUIRE(a.reset_buf != nullptr || a.env_ids_in != nullptr, "%s: neither a reset mask nor an env id list", who);
  PULSE_REQUIRE(a.env_ids_in == nullptr || (a.num_ids >= 0 && a.num_ids <= num_envs), "%s: num_ids %lld outside [0, %lld]", who,
                (long long)a.num_ids, (long long)num_envs);
  PULSE_REQUIRE(a.env_list != nullptr && a.count != nullptr, "%s: env_list / count outputs are required", who);
  PULSE_REQUIRE(a.motion_ids && a.motion_start_times && a.motion_start_offset && a.global_offset && a.progress_buf, "%s: null task buffer", who);
  PULSE_REQUIRE(a.root_states && a.dof_pos && a.dof_vel, "%s: null simulator tensor", who);
  PULSE_REQUIRE(a.root_env_stride >= PULSE_BODY_STATE_W && a.dof_elem_stride >= 1 && a.dof_env_stride >= PULSE_NUM_DOF * a.dof_elem_stride,
                "%s: bad root / dof strides", who);
  PULSE_REQUIRE(a.rigid_body_state == nullptr || a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "%s: body_env_stride too small", who);
  PULSE_REQUIRE(a.contact_forces == nullptr || (a.contact_bodies >= 0 && a.contact_env_stride >= 3 * a.contact_bodies),
                "%s: bad contact-force strides", who);
  PULSE_REQUIRE(a.amp_obs_buf == nullptr || (a.num_amp_steps >= 1 && a.num_amp_steps <= 16), "%s: num_amp_steps outside [1,16]", who);
  PULSE_REQUIRE(lib->d.aux_rec != nullptr, "%s: the MotionLib handle has no aux records (dof_pos / dof_vel)", who);
  return PULSE_OK;
}

// reset_ref_state_kernel over a.env_list[0 .. *a.count), at most `upper_envs` envs: a persistent grid that strides over the
// device-side count.
inline int launch_ref_state(const pulse_motionlib_t* lib, const pulse_reset_args_t& a, long long upper_envs, cudaStream_t st) {
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0;
    PULSE_CUDA_OK(cudaGetDevice(&dev));
    PULSE_CUDA_OK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const int steps = a.amp_obs_buf != nullptr ? a.num_amp_steps : 1;
  const long long upper = upper_envs * steps;                                                 // warps if every env were reset
  long long blocks = (upper + 7) / 8;
  if (blocks > num_sms * 8) blocks = num_sms * 8;
  if (blocks < 1) blocks = 1;
  reset_ref_state_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(lib->d, a);
  PULSE_LAUNCH_OK("reset_ref_state_kernel");
  return PULSE_OK;
}

}  // namespace pulse
