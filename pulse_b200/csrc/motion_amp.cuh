// The reference-motion pieces shared by the resets (reset_warps.cuh) and the AMP demo fetch (amp_buffers.cu): the clip and start-time
// draws of MotionLibBase (sample_motions, sample_time_interval) and the AMP observation of the un-adjusted motion in either body layout.
#pragma once
#include "humanoid_obs.cuh"

namespace pulse {
namespace {

// sample_motions: the first clip whose inclusive CDF exceeds u * total (a zero-weight clip never does before its predecessor).
__device__ __forceinline__ long long pick_motion(const float* cdf, long long m, float u) {
  const float total = cdf[m - 1];
  float v = __fmul_rn(u, total);
  if (v >= total) v = nextafterf(total, 0.0f);
  long long lo = 0, hi = m - 1;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (cdf[mid] > v) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// sample_time_interval (motion_lib_base.py:411-420): ((phase * motion_len) / curr_fps).long() * curr_fps with curr_fps = 1/30.
__device__ __forceinline__ float sample_time_interval(float phase, float mlen) {
  const float step30 = static_cast<float>(1.0 / 30.0);
  return __fmul_rn(__ll2float_rn(static_cast<long long>(__fdiv_rn(__fmul_rn(phase, mlen), step30))), step30);
}

// build_amp_observations_smpl in body layout L into the warp's staging row (L::kAmpObs floats), then `width` floats of it to `out`:
// L::kAmpObs is the whole row, one less drops the root height.  A non-upright start takes the heading and root rotation feature of
// remove_base_rot(q0).
template <class L = SmplLayout, class JointFn, class KeyPosFn>
__device__ __forceinline__ void store_amp_row(float* out, int width, float* stage, int lane, Vec3 p0, Quat q0, Vec3 v0, Vec3 w0, bool upright,
                                              JointFn joint, KeyPosFn key_pos) {
  store_amp_obs<L>(stage, lane, p0, base_rot_removed(q0, upright), v0, w0, joint, key_pos);
  __syncwarp();
  const int skip = L::kAmpObs - width;
  for (int c = lane; c < width; c += 32) out[c] = stage[skip + c];
  __syncwarp();
}

// The AMP row of the layout-L motion blended between the frame records r0p / r1p (aux records x0 / x1) at weight b, as it is:
// without the ground fix or a pose adjustment (_init_amp_obs_ref, build_amp_obs_demo).  Record offsets for B bodies: frame pos 0,
// rot 3B, vel 7B, ang vel 10B; aux local rotations 0 (joint jt at body jt + 1), dof velocities 4B.
template <class L = SmplLayout>
__device__ __forceinline__ void store_motion_amp_row(float b, const float* r0p, const float* r1p,
                                                     const float* x0, const float* x1, float* out, int width, float* stage, int lane,
                                                     bool upright) {
  constexpr int B = L::kBodies, kRot = 3 * B, kVel = 7 * B, kAng = 10 * B, kDvs = 4 * B;
  const Vec3 p0 = {lerp_rn(r0p[0], r1p[0], b), lerp_rn(r0p[1], r1p[1], b), lerp_rn(r0p[2], r1p[2], b)};
  const Vec3 v0 = {lerp_rn(r0p[kVel], r1p[kVel], b), lerp_rn(r0p[kVel + 1], r1p[kVel + 1], b), lerp_rn(r0p[kVel + 2], r1p[kVel + 2], b)};
  const Vec3 w0 = {lerp_rn(r0p[kAng], r1p[kAng], b), lerp_rn(r0p[kAng + 1], r1p[kAng + 1], b), lerp_rn(r0p[kAng + 2], r1p[kAng + 2], b)};
  const Quat q0 = slerp(ldq4(r0p + kRot), ldq4(r1p + kRot), b);
  const auto joint = [&](int jt) {
    return AmpJoint{quat_exp_map(slerp(ldq4(x0 + 4 * (jt + 1)), ldq4(x1 + 4 * (jt + 1)), b)),
                    {lerp_rn(x0[kDvs + 3 * jt], x1[kDvs + 3 * jt], b), lerp_rn(x0[kDvs + 1 + 3 * jt], x1[kDvs + 1 + 3 * jt], b),
                     lerp_rn(x0[kDvs + 2 + 3 * jt], x1[kDvs + 2 + 3 * jt], b)}};
  };
  const auto key_pos = [&](int kb) {
    return Vec3{lerp_rn(r0p[3 * kb], r1p[3 * kb], b), lerp_rn(r0p[3 * kb + 1], r1p[3 * kb + 1], b), lerp_rn(r0p[3 * kb + 2], r1p[3 * kb + 2], b)};
  };
  store_amp_row<L>(out, width, stage, lane, p0, q0, v0, w0, upright, joint, key_pos);
}

}  // namespace
}  // namespace pulse
