// The per-warp reference-state reset shared by pulse_reset_ztask (ztask_reset.cu) and pulse_reset_terrain (terrain_reset.cu):
//   reset_compact_kernel  one CTA: the ordered compaction of compact.cuh turns the reset mask or id list into the ascending env list,
//                         the humanoid and target actor lists and a device-side count;
//   reset_warps           one warp per (reset env, AMP history step k), for a body layout (SMPL, SMPL-X): clip and start-time
//                         draws, MotionLib gather, SMPL ground fix from the per-frame floor table, the caller's adjustment of the root
//                         and bodies, the scatter into the simulator's views, counters and the AMP rows (195 / 196 floats for SMPL, 465 / 466 for SMPL-X).
// The entry points, argument structs and Philox word layout are documented in include/pulse_b200.h.
#pragma once
#include "compact.cuh"
#include "motion_amp.cuh"
#include "philox.cuh"

namespace pulse {
namespace {

constexpr int kResetWarps = 8;

__global__ void __launch_bounds__(kCompactThreads) reset_compact_kernel(const pulse_ztask_reset_args_t a, long long num_envs) {
  __shared__ int warp_cnt[kCompactThreads / 32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const long long n = a.env_ids_in != nullptr ? a.num_ids : num_envs;
  for (long long c0 = 0; c0 < n; c0 += kCompactThreads) {
    const long long i = c0 + threadIdx.x;
    long long env = -1;
    if (i < n && a.env_ids_in == nullptr) env = a.reset_buf[i] != 0 ? i : -1;
    if (i < n && a.env_ids_in != nullptr) {   // an id outside [0, N) or not above its predecessor is skipped: each env is written once
      env = a.env_ids_in[i];
      if (env < 0 || env >= num_envs || (i > 0 && a.env_ids_in[i - 1] >= env)) env = -1;
    }
    const int pos = compact_slot(env >= 0, warp_cnt, &base);
    if (pos < 0) continue;
    a.env_list[pos] = env;
    if (a.actor_list != nullptr) a.actor_list[pos] = a.actor_ids != nullptr ? a.actor_ids[env] : static_cast<int>(env);
    if (a.tar_actor_list != nullptr) a.tar_actor_list[pos] = a.tar_actor_ids != nullptr ? a.tar_actor_ids[env] : static_cast<int>(env);
    if (a.amp_fresh != nullptr) a.amp_fresh[env] = 1;
  }
  if (threadIdx.x == 0) *a.count = base;
}

// The work of one warp in body layout L (lib: the layout's MotionLib descriptor).  `adjust(e, lane, r0, off, p, rq, v, rp, rr, rv, rw)`
// runs after the ground fix once per body a lane holds (lane l holds bodies l and l + 32 where the layout has them): (p, rq, v) are
// that body's position, rotation and velocity, (rp, rr, rv, rw) the root's in every lane; a lane's second call gets its own copy of the
// root, so the root is adjusted once.  r0 is Philox block (seed, e, off) when a draw is not injected or `more_draws` is set, zero
// otherwise.  What it leaves is what _set_env_state writes.  The AMP history rows are layout L's (`stage`: L::kAmpObs floats).
template <class L, class Lib, class Adjust>
__device__ __forceinline__ void reset_warps(const Lib& lib, const pulse_ztask_reset_args_t& a, bool more_draws, float* stage,
                                            const Adjust& adjust) {
  constexpr int B = L::kBodies, kSlots = (B + 31) / 32;
  constexpr int kRot = 3 * B, kVel = 7 * B, kAng = 10 * B, kDvs = 4 * B;   // record offsets
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int steps = a.amp_obs_buf != nullptr ? a.num_amp_steps : 1;
  const long long items = static_cast<long long>(*a.count) * steps;
  const unsigned long long off = a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull);
  const bool upright = a.upright != 0;
  for (long long it = warp0; it < items; it += nwarps) {
    const long long i = it / steps;
    const int k = static_cast<int>(it - i * steps);
    const long long e = a.env_list[i];
    Philox4 r0{0u, 0u, 0u, 0u};
    if ((a.motion_ids_in == nullptr && a.motion_u == nullptr) || a.phase == nullptr || more_draws)
      r0 = philox4x32_10(a.seed, static_cast<unsigned long long>(e), off);
    const long long mid = a.motion_ids_in != nullptr ? a.motion_ids_in[e]
                          : pick_motion(a.sampling_cdf, lib.num_motions, a.motion_u != nullptr ? a.motion_u[e] : u01(r0.y));
    const float mlen = lib.lengths[mid];
    float t0 = 0.0f;
    if (a.state_init == PULSE_ZINIT_RANDOM) {   // sample_time_interval: ((phase * motion_len) / curr_fps).long() * curr_fps
      const float ph = a.phase != nullptr ? a.phase[e] : u01(r0.x);
      t0 = sample_time_interval(ph, mlen);
    }
    const float t = k == 0 ? t0 : __fadd_rn(t0, __fmul_rn(-a.dt, static_cast<float>(k)));
    long long i0, i1;
    float b;
    frame_blend_rn(t, mlen, lib.num_frames[mid], lib.dt[mid], i0, i1, b);
    const long long f0 = i0 + lib.length_starts[mid], f1 = i1 + lib.length_starts[mid];
    const float* r0p = lib.frame_rec + f0 * L::kFrameRec;
    const float* r1p = lib.frame_rec + f1 * L::kFrameRec;
    const float* x0 = lib.aux_rec + f0 * L::kAuxRec;
    const float* x1 = lib.aux_rec + f1 * L::kAuxRec;

    if (k > 0) {   // _init_amp_obs_ref: the motion at t0 - k dt as it is, without the ground fix or the pose adjustment
      store_motion_amp_row<L>(b, r0p, r1p, x0, x1, a.amp_obs_buf + (e * a.num_amp_steps + k) * a.amp_width, a.amp_width, stage, lane,
                              upright);
      continue;
    }

    // ---- the reset state: lane l holds bodies l (slot 0) and l + 32 (slot 1) -------------------------------------------------------
    Vec3 p[kSlots], v[kSlots], w[kSlots];
    Quat rq[kSlots];
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
      const int j = lane + 32 * s < B ? lane + 32 * s : 0;
      p[s] = {lerp_rn(r0p[3 * j], r1p[3 * j], b), lerp_rn(r0p[3 * j + 1], r1p[3 * j + 1], b), lerp_rn(r0p[3 * j + 2], r1p[3 * j + 2], b)};
      v[s] = {lerp_rn(r0p[kVel + 3 * j], r1p[kVel + 3 * j], b), lerp_rn(r0p[kVel + 1 + 3 * j], r1p[kVel + 1 + 3 * j], b),
              lerp_rn(r0p[kVel + 2 + 3 * j], r1p[kVel + 2 + 3 * j], b)};
      w[s] = {lerp_rn(r0p[kAng + 3 * j], r1p[kAng + 3 * j], b), lerp_rn(r0p[kAng + 1 + 3 * j], r1p[kAng + 1 + 3 * j], b),
              lerp_rn(r0p[kAng + 2 + 3 * j], r1p[kAng + 2 + 3 * j], b)};
      rq[s] = slerp(ldq4(r0p + kRot + 4 * j), ldq4(r1p + kRot + 4 * j), b);
    }
    // ground fix (humanoid_amp.py:382-430): d = min_v (V - (J0 - root)).z - 0.02 = (floor(f0) + root z) - 0.02
    const float root_z = __shfl_sync(kFull, p[0].z, 0);
    const float d = __fsub_rn(__fadd_rn(a.floor[f0], root_z), 0.02f);
#pragma unroll
    for (int s = 0; s < kSlots; ++s) p[s].z = __fsub_rn(p[s].z, d);
    Vec3 rp = {__shfl_sync(kFull, p[0].x, 0), __shfl_sync(kFull, p[0].y, 0), __shfl_sync(kFull, p[0].z, 0)};
    Quat rr = {__shfl_sync(kFull, rq[0].x, 0), __shfl_sync(kFull, rq[0].y, 0), __shfl_sync(kFull, rq[0].z, 0), __shfl_sync(kFull, rq[0].w, 0)};
    Vec3 rv = {__shfl_sync(kFull, v[0].x, 0), __shfl_sync(kFull, v[0].y, 0), __shfl_sync(kFull, v[0].z, 0)};
    Vec3 rw = {__shfl_sync(kFull, w[0].x, 0), __shfl_sync(kFull, w[0].y, 0), __shfl_sync(kFull, w[0].z, 0)};
#pragma unroll
    for (int s = kSlots - 1; s >= 1; --s) {   // the later slots first, on copies of the root the slot-0 call then adjusts
      Vec3 cp = rp, cv = rv, cw = rw;
      Quat cr = rr;
      adjust(e, lane, r0, off, p[s], rq[s], v[s], cp, cr, cv, cw);
    }
    adjust(e, lane, r0, off, p[0], rq[0], v[0], rp, rr, rv, rw);
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
      const int j = lane + 32 * s;
      if (j < B) {   // _set_env_state (humanoid_amp.py:565-597)
        float* bs = a.rigid_body_state + e * a.body_env_stride + j * PULSE_BODY_STATE_W;
        bs[0] = p[s].x; bs[1] = p[s].y; bs[2] = p[s].z; bs[3] = rq[s].x; bs[4] = rq[s].y; bs[5] = rq[s].z; bs[6] = rq[s].w;
        bs[7] = v[s].x; bs[8] = v[s].y; bs[9] = v[s].z; bs[10] = w[s].x; bs[11] = w[s].y; bs[12] = w[s].z;
        if (j >= 1) {   // dof_pos = exp_map(slerp(local rotations)) of joints 1..B-1
          const Vec3 em = quat_exp_map(slerp(ldq4(x0 + 4 * j), ldq4(x1 + 4 * j), b));
          float* dp = a.dof_pos + e * a.dof_env_stride + 3 * (j - 1) * a.dof_elem_stride;
          dp[0] = em.x; dp[a.dof_elem_stride] = em.y; dp[2 * a.dof_elem_stride] = em.z;
        }
      }
    }
    for (int c = lane; c < L::kDofs; c += 32) a.dof_vel[e * a.dof_env_stride + c * a.dof_elem_stride] = lerp_rn(x0[kDvs + c], x1[kDvs + c], b);
    if (a.contact_forces != nullptr)
      for (int c = lane; c < a.contact_bodies * 3; c += 32) a.contact_forces[e * a.contact_env_stride + c] = 0.0f;
    if (lane == 0) {
      float* rs = a.root_states + e * a.root_env_stride;
      rs[0] = rp.x; rs[1] = rp.y; rs[2] = rp.z; rs[3] = rr.x; rs[4] = rr.y; rs[5] = rr.z; rs[6] = rr.w;
      rs[7] = rv.x; rs[8] = rv.y; rs[9] = rv.z; rs[10] = rw.x; rs[11] = rw.y; rs[12] = rw.z;
      a.sampled_motion_ids[e] = mid;   // humanoid_amp.py:484-485
      a.motion_start_times[e] = t0;
      a.progress_buf[e] = 0;           // _reset_env_tensors (humanoid.py:603-606)
      if (a.reset_buf != nullptr) a.reset_buf[e] = 0;
      if (a.terminate_buf != nullptr) a.terminate_buf[e] = 0;
    }
    if (a.amp_obs_buf == nullptr) continue;
    // row 0: _compute_amp_observations(env_ids) of the rigid bodies and dofs just written
    __syncwarp();
    const float* bs = a.rigid_body_state + e * a.body_env_stride;
    const float* dp = a.dof_pos + e * a.dof_env_stride;
    const float* dv = a.dof_vel + e * a.dof_env_stride;
    const long long ds = a.dof_elem_stride;
    const auto joint = [&](int jt) {
      return AmpJoint{{dp[(3 * jt + 0) * ds], dp[(3 * jt + 1) * ds], dp[(3 * jt + 2) * ds]},
                      {dv[(3 * jt + 0) * ds], dv[(3 * jt + 1) * ds], dv[(3 * jt + 2) * ds]}};
    };
    const auto key_pos = [&](int kb) { return ldv(bs + kb * PULSE_BODY_STATE_W); };
    store_amp_row<L>(a.amp_obs_buf + e * a.num_amp_steps * a.amp_width, a.amp_width, stage, lane, ldv(bs), ldq(bs + 3), ldv(bs + 7), ldv(bs + 10),
                     upright, joint, key_pos);
  }
}

}  // namespace
}  // namespace pulse
