// Heightfield sampling of the pedestrian terrain task, shared by the step, height and spawn-reset kernels (terrain.cu,
// terrain_reset.cu): Terrain.world_points_to_map / sample_height_points (humanoid_pedestrian_terrain.py:1191-1198, :1261-1267) and
// get_center_heights (:690-716).  Cell indices are integers decided by fp32 arithmetic, so the operations that feed them keep the
// reference's order with round-to-nearest intrinsics (no FMA contraction).
#pragma once
#include "humanoid_obs.cuh"

namespace pulse {

// isaacgym.torch_utils.quat_apply [3P-memory]: t = 2 (xyz x b); b + w t + xyz x t, in this order.
__device__ __forceinline__ Vec3 cross_rn(Vec3 a, Vec3 b) {
  return {__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)), __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
          __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
__device__ __forceinline__ Vec3 quat_apply_rn(Quat q, Vec3 b) {
  const Vec3 u = {q.x, q.y, q.z};
  Vec3 t = cross_rn(u, b);
  t = {__fmul_rn(t.x, 2.0f), __fmul_rn(t.y, 2.0f), __fmul_rn(t.z, 2.0f)};
  const Vec3 c = cross_rn(u, t);
  return {__fadd_rn(__fadd_rn(b.x, __fmul_rn(q.w, t.x)), c.x), __fadd_rn(__fadd_rn(b.y, __fmul_rn(q.w, t.y)), c.y),
          __fadd_rn(__fadd_rn(b.z, __fmul_rn(q.w, t.z)), c.z)};
}

// quat_apply_yaw (:1571-1576): x = y = 0, normalize, quat_apply
__device__ __forceinline__ Quat yaw_only(Quat q) {
  const float n = fmaxf(__fsqrt_rn(__fadd_rn(__fmul_rn(q.z, q.z), __fmul_rn(q.w, q.w))), 1e-9f);
  return {0.0f, 0.0f, __fdiv_rn(q.z, n), __fdiv_rn(q.w, n)};
}

struct HeightField {
  const int16_t* hf;
  long long rows, cols;
  float hscale, vscale;
};

// Terrain.world_points_to_map + sample_height_points (:1191-1198, :1261-1267): long(x / horizontal_scale) truncates toward zero,
// the indices clip to [0, dim - 2], height = min(hf[px, py], hf[px + 1, py + 1]) * vertical_scale.  A plane (hf == NULL) is flat 0.
__device__ __forceinline__ float sample_height(const HeightField& t, float x, float y) {
  if (t.hf == nullptr) return 0.0f;
  long long px = static_cast<long long>(__fdiv_rn(x, t.hscale));
  long long py = static_cast<long long>(__fdiv_rn(y, t.hscale));
  px = min(max(px, 0ll), t.rows - 2);
  py = min(max(py, 0ll), t.cols - 2);
  const int h1 = __ldg(t.hf + px * t.cols + py), h2 = __ldg(t.hf + (px + 1) * t.cols + py + 1);
  return __fmul_rn(static_cast<float>(min(h1, h2)), t.vscale);
}

// world point = quat_apply(q, offset) + origin (get_heights :734-742, get_center_heights :703-711)
__device__ __forceinline__ float height_at(const HeightField& t, Quat q, const float* off, Vec3 origin) {
  const Vec3 r = quat_apply_rn(q, Vec3{off[0], off[1], off[2]});
  return sample_height(t, __fadd_rn(r.x, origin.x), __fadd_rn(r.y, origin.y));
}

// mean of get_center_heights over the points (lanes < count hold one point each); the result is in every lane
__device__ __forceinline__ float center_height(const HeightField& t, const float* pts, int count, Quat q_root, Vec3 p_root, bool upright,
                                               int lane) {
  const Quat qy = yaw_only(base_rot_removed(q_root, upright));
  float h = 0.0f;
  for (int i = lane; i < count; i += 32) h += height_at(t, qy, pts + 3 * i, p_root);
  return warp_sum(h) / static_cast<float>(count);
}

}  // namespace pulse
