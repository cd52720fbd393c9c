// Task observation of HumanoidIm for EVERY observation version / tracked-body subset / number of future samples (SURVEY 8f-4):
// one launch replaces `_compute_task_obs`'s dispatch over compute_imitation_observations, _v2, _v3, _v6, _v7, _v8, _v9
// (phc/env/tasks/humanoid_im.py:757-833, :1222-1540).  The fused step kernel (im_step.cu) stays specialised for the default
// configuration (obs_v 6, 24 bodies, one sample); this kernel is the general skeleton: one warp per env, the (sample, body) items of
// the env spread over its lanes, every item computing only the features its version asks for and storing them at the offset the
// reference's concatenation gives them.  Reference states come from pulse_motion_state on the env's `time_steps` sample times, in
// the reference's repeat_interleave order (row env * T + t).
#include "pulse_common.cuh"
#include "quat_math.cuh"

namespace pulse {
namespace {

__global__ void __launch_bounds__(128) task_obs_kernel(const pulse_task_obs_args_t a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= a.num_envs) return;
  const long long e = warp;
  const int J = a.num_track, T = a.time_steps, V = a.version;
  const float* bs = a.body_state + e * a.body_env_stride;
  // heading of the ROOT body (body 0 of the env, not of the subset): humanoid_im.py:746-747
  const Vec3 p_root = ldv(bs);
  const Quat q_root = base_rot_removed(ldq(bs + 3), a.upright != 0);
  float hs, hc;
  heading_half(q_root, hs, hc);
  const Yaw yr = make_yaw(Quat{0.0f, 0.0f, -hs, hc});
  float* o = a.obs + e * a.obs_stride;
  const int TJ = T * J;
  for (int it = lane; it < TJ; it += 32) {
    const int t = it / J, j = it - t * J;
    const int b = a.track_ids[j];
    const float* s = bs + b * PULSE_BODY_STATE_W;
    const Vec3 p = ldv(s), v = ldv(s + 7), w = ldv(s + 10);
    const Quat q = ldq(s + 3);
    const long long r = (e * T + t) * PULSE_NUM_BODIES + b;          // row of the reference arrays
    const Vec3 rp = ldv(a.ref_pos + r * 3);
    const Vec3 d_pos = yaw_rot(yr, rp - p);
    if (V == 7) {                                                    // :1381-1413   per t: [dp | dv | R(pref - root)]
      float* ot = o + t * (9 * J);
      stv(ot + 3 * j, d_pos);
      stv(ot + 3 * J + 3 * j, yaw_rot(yr, ldv(a.ref_vel + r * 3) - v));
      stv(ot + 6 * J + 3 * j, yaw_rot(yr, rp - p_root));
      continue;
    }
    const Quat rq = ldq(a.ref_rot + r * 4);
    float d_rot[6];
    qsix(yaw_mul_right(yaw_mul_left(-hs, hc, qmul(rq, qconj(q))), hs, hc), d_rot);
    if (V == 1 || V == 2 || V == 3) {                                // :1222-1326   flat blocks over (t, j)
      stv(o + 3 * it, d_pos);
#pragma unroll
      for (int k = 0; k < 6; ++k) o[3 * TJ + 6 * it + k] = d_rot[k];
      if (V != 3) {
        stv(o + 9 * TJ + 3 * it, yaw_rot(yr, ldv(a.ref_vel + r * 3) - v));
        stv(o + 12 * TJ + 3 * it, yaw_rot(yr, ldv(a.ref_ang_vel + r * 3) - w));
      }
      if (V == 2 && j >= 1) {                                        // :1296-1298  dof difference of the tracked joints (T = 1)
        const int d0 = 3 * (b - 1);
        const float* dp = a.dof_pos + e * a.dof_env_stride;
        const float* rd = a.ref_dof_pos + e * PULSE_NUM_DOF;
#pragma unroll
        for (int k = 0; k < 3; ++k) o[15 * TJ + 3 * (j - 1) + k] = rd[d0 + k] - dp[(d0 + k) * a.dof_elem_stride];
      }
      continue;
    }
    float l_rot[6];
    qsix(yaw_mul_left(-hs, hc, rq), l_rot);
    const Vec3 l_pos = yaw_rot(yr, rp - p_root);
    if (V == 6) {                                                    // :1328-1378   per t: [dp | drot | dv | dw | lp | lrot]
      float* ot = o + t * (24 * J);
      stv(ot + 3 * j, d_pos);
#pragma unroll
      for (int k = 0; k < 6; ++k) ot[3 * J + 6 * j + k] = d_rot[k];
      stv(ot + 9 * J + 3 * j, yaw_rot(yr, ldv(a.ref_vel + r * 3) - v));
      stv(ot + 12 * J + 3 * j, yaw_rot(yr, ldv(a.ref_ang_vel + r * 3) - w));
      stv(ot + 15 * J + 3 * j, l_pos);
#pragma unroll
      for (int k = 0; k < 6; ++k) ot[18 * J + 6 * j + k] = l_rot[k];
    } else if (V == 8) {                                             // :1415-1479, time_steps = 1 branch (:1472-1476)
      const Vec3 rv = ldv(a.ref_vel + r * 3), rw = ldv(a.ref_ang_vel + r * 3);
      stv(o + 3 * j, d_pos);
#pragma unroll
      for (int k = 0; k < 6; ++k) o[3 * J + 6 * j + k] = d_rot[k];
      stv(o + 9 * J + 3 * j, yaw_rot(yr, rv - v));
      stv(o + 12 * J + 3 * j, yaw_rot(yr, rw - w));
      stv(o + 15 * J + 3 * j, l_pos);
#pragma unroll
      for (int k = 0; k < 6; ++k) o[18 * J + 6 * j + k] = l_rot[k];
      stv(o + 24 * J + 3 * j, yaw_rot(yr, rv));
      stv(o + 27 * J + 3 * j, yaw_rot(yr, rw));
    } else {                                                         // 9  :1482-1540  per t: [dp | drot | d root v | d root w | lp | lrot]
      float* ot = o + t * (18 * J + 6);
      stv(ot + 3 * j, d_pos);
#pragma unroll
      for (int k = 0; k < 6; ++k) ot[3 * J + 6 * j + k] = d_rot[k];
      if (j == 0) {   // root = tracked body 0 (ref_body_vel_subset[:, 0], body_vel[:, 0]; humanoid_im.py:800-802)
        stv(ot + 9 * J, yaw_rot(yr, ldv(a.ref_vel + r * 3) - v));
        stv(ot + 9 * J + 3, yaw_rot(yr, ldv(a.ref_ang_vel + r * 3) - w));
      }
      stv(ot + 9 * J + 6 + 3 * j, l_pos);
#pragma unroll
      for (int k = 0; k < 6; ++k) ot[12 * J + 6 + 6 * j + k] = l_rot[k];
    }
  }
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_task_obs_size(int32_t version, int32_t num_track, int32_t time_steps) {
  const int J = num_track, T = time_steps;
  switch (version) {
    case 1: return 15 * T * J;
    case 2: return 15 * J + 3 * (J - 1);
    case 3: return 9 * T * J;
    case 6: return 24 * T * J;
    case 7: return 9 * T * J;
    case 8: return 30 * J;
    case 9: return T * (18 * J + 6);
    default: return -1;
  }
}

extern "C" int pulse_im_task_obs(const pulse_task_obs_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_im_task_obs: null args");
  const pulse_task_obs_args_t& a = *args;
  const int size = pulse_task_obs_size(a.version, a.num_track, a.time_steps);
  PULSE_REQUIRE(size > 0, "pulse_im_task_obs: unsupported observation version %d", a.version);
  PULSE_REQUIRE(a.num_envs > 0 && a.num_track >= 1 && a.num_track <= PULSE_NUM_BODIES && a.time_steps >= 1,
                "pulse_im_task_obs: num_envs %lld, num_track %d, time_steps %d", (long long)a.num_envs, a.num_track, a.time_steps);
  PULSE_REQUIRE(a.time_steps == 1 || (a.version != 2 && a.version != 8),
                "pulse_im_task_obs: versions 2 and 8 are built for time_steps = 1 (the reference's multi-sample branches of these index a flattened tensor by column)");
  PULSE_REQUIRE(a.body_state && a.track_ids && a.ref_pos && a.obs, "pulse_im_task_obs: null buffer");
  PULSE_REQUIRE(a.version == 7 || a.ref_rot != nullptr, "pulse_im_task_obs: ref_rot is null");
  PULSE_REQUIRE(a.version == 3 || a.ref_vel != nullptr, "pulse_im_task_obs: ref_vel is null");
  PULSE_REQUIRE(a.version == 3 || a.version == 7 || a.ref_ang_vel != nullptr, "pulse_im_task_obs: ref_ang_vel is null");
  PULSE_REQUIRE(a.version != 2 || (a.dof_pos && a.ref_dof_pos && a.dof_elem_stride >= 1), "pulse_im_task_obs: version 2 needs dof_pos / ref_dof_pos");
  PULSE_REQUIRE(a.obs_stride >= size, "pulse_im_task_obs: obs_stride %lld < %d", (long long)a.obs_stride, size);
  PULSE_REQUIRE(a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "pulse_im_task_obs: body_env_stride %lld < 312", (long long)a.body_env_stride);
  const int warps = 4;
  task_obs_kernel<<<static_cast<unsigned>((a.num_envs + warps - 1) / warps), warps * 32, 0, static_cast<cudaStream_t>(stream)>>>(a);
  PULSE_LAUNCH_OK("task_obs_kernel");
  return PULSE_OK;
}
