// One env of the latent-space tasks' post-physics step (the SMPL reach, speed and strike tasks; the SMPL-X speed, reach and strike
// tasks), one warp per env, lane = body: self observation, task observation, reward and reset.  ztask_kernel (ztask_step.cu) runs it
// in its step, list-observation and rollout modes, so all of them produce the same rows bit for bit.
#pragma once
#include "humanoid_obs.cuh"

namespace pulse {

// One env of the step in body layout L (SmplReachLayout: reach; SmplLayout: speed and strike; SmplxLayout: speed; SmplxTargetLayout:
// reach and strike).  kObsOnly: the observation alone.  Lane l holds bodies l and l + 32 (the second only where the layout has more than 32 bodies).
// ztask_is<L, K>: whether env work takes task kind K's branch -- a constant where the layout serves K alone or not at all.
template <class L, int K>
constexpr bool kServes = (L::kTasks >> K) & 1u;
template <class L, int K>
__device__ __forceinline__ bool ztask_is(const typename L::StepArgs& a) {
  if constexpr (!kServes<L, K>) return false;
  else if constexpr (L::kTasks == (1u << K)) return true;
  else return a.kind == K;
}

template <class L, bool kObsOnly>
__device__ __forceinline__ void ztask_env(const typename L::StepArgs& a, long long e, int lane) {
  constexpr int kSlots = (L::kBodies + 31) / 32;
  Vec3 p[kSlots], v[kSlots], w[kSlots];
  Quat q[kSlots];
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    const int j = lane + 32 * s;
    const float* bs = a.body_state + e * a.body_env_stride + (j < L::kBodies ? j : 0) * 13;
    p[s] = {bs[0], bs[1], bs[2]};
    v[s] = {bs[7], bs[8], bs[9]};
    w[s] = {bs[10], bs[11], bs[12]};
    q[s] = {bs[3], bs[4], bs[5], bs[6]};
  }
  const Vec3 p_root = {__shfl_sync(kFull, p[0].x, 0), __shfl_sync(kFull, p[0].y, 0), __shfl_sync(kFull, p[0].z, 0)};
  const Quat q_root = {__shfl_sync(kFull, q[0].x, 0), __shfl_sync(kFull, q[0].y, 0), __shfl_sync(kFull, q[0].z, 0), __shfl_sync(kFull, q[0].w, 0)};
  float hs, hc;
  heading_half(q_root, hs, hc);
  const Yaw yr = make_yaw(Quat{0.0f, 0.0f, -hs, hc});
  // the self observation's heading: the root's own (upright start) or that of remove_base_rot(root) (humanoid.py:1682-1684); the
  // task observation below keeps the root's own either way (compute_speed_observations reads the raw root rotation)
  float shs = hs, shc = hc;
  Yaw syr = yr;
  if constexpr (!L::kUpright) {
    heading_half(base_rot_removed(q_root, false), shs, shc);
    syr = make_yaw(Quat{0.0f, 0.0f, -shs, shc});
  }
  float* o = a.obs_buf + e * a.obs_stride;
  bool contact = false, height = false, hard_contact = false;
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    const int j = lane + 32 * s;
    const bool body = j < L::kBodies;
    if (body) store_self_obs<L::kBodies>(o, j, p[s], p_root, q[s], v[s], w[s], shs, shc, syr);
    const FallFlags fall = fall_flags(a, e, j, body, p[s].z);
    contact = contact || fall.contact;
    height = height || fall.height;
    if constexpr (kServes<L, PULSE_ZTASK_STRIKE>) {
      // strike: a body that is neither a ground-contact body nor a strike body pressing harder than 50 N (humanoid_strike.py:356-364)
      if (a.enable_early_termination && body && a.contact_forces != nullptr && !(((a.contact_body_mask | a.strike_body_mask) >> j) & 1u)) {
        const float* cf = a.contact_forces + e * a.contact_env_stride + j * 3;
        hard_contact = hard_contact || fabsf(cf[0]) > 50.0f || fabsf(cf[1]) > 50.0f || fabsf(cf[2]) > 50.0f;
      }
    }
  }
  const bool any_contact = __any_sync(kFull, contact), any_height = __any_sync(kFull, height);
  bool any_hard = false;
  float power = 0.0f;
  if constexpr (kServes<L, PULSE_ZTASK_STRIKE>) any_hard = __any_sync(kFull, hard_contact);
  if constexpr (L::kPower) {
    // power term of the speed task: -c * sum |tau * qdot|, zero for progress <= 3 (humanoid_speed.py:215-222)
    power = a.kind == PULSE_ZTASK_SPEED && a.dof_force != nullptr ? dof_power(a, e, lane) : 0.0f;
  }
  // reach: the reach body's position, broadcast from its slot and lane (a shuffle every lane takes part in)
  Vec3 p_reach = {0.0f, 0.0f, 0.0f};
  if constexpr (kServes<L, PULSE_ZTASK_REACH> && !kObsOnly) {
    if (ztask_is<L, PULSE_ZTASK_REACH>(a)) {
      const int rs = a.reach_body_id >> 5, rl = a.reach_body_id & 31;
      Vec3 src = p[0];
#pragma unroll
      for (int s = 1; s < kSlots; ++s)
        if (s == rs) src = p[s];
      p_reach = {__shfl_sync(kFull, src.x, rl), __shfl_sync(kFull, src.y, rl), __shfl_sync(kFull, src.z, rl)};
    }
  }
  if (lane == 0) {
    const long long prog = kObsOnly ? 0 : a.progress_buf[e];
    float vx = 0.0f, vy = 0.0f;
    if constexpr (!kObsOnly && L::kTasks != (1u << PULSE_ZTASK_REACH)) {   // the SMPL reach struct has no prev_root_pos and no dt
      if (!ztask_is<L, PULSE_ZTASK_REACH>(a)) {
        const float* pr = a.prev_root_pos + 3 * e;
        vx = (p_root.x - pr[0]) / a.dt;                                            // root_vel = delta_root_pos / dt
        vy = (p_root.y - pr[1]) / a.dt;
      }
    }
    float* t = o + L::kSelfObs;
    bool failed = any_contact && any_height;
    if (ztask_is<L, PULSE_ZTASK_SPEED>(a)) {
      if constexpr (kServes<L, PULSE_ZTASK_SPEED>) {
        // observation: heading-frame x axis (first two components) and the target speed (:310-325)
        const Vec3 d = yaw_rot(yr, Vec3{1.0f, 0.0f, 0.0f});
        const float ts = a.tar_speed[e];
        t[0] = d.x; t[1] = d.y; t[2] = ts;
        if constexpr (kObsOnly) return;
        const float err = ts - vx;
        float rew = expf(-0.25f * (err * err + 0.1f * vy * vy));                    // :327-343
        if (a.reward_raw != nullptr) a.reward_raw[e * a.raw_stride] = rew;
        if constexpr (L::kPower) {
          if (a.dof_force != nullptr) {
            const float pw = prog <= 3 ? 0.0f : -a.power_coefficient * power;
            rew += pw;
            if (a.reward_raw != nullptr) a.reward_raw[e * a.raw_stride + 1] = pw;
          }
        }
        a.rew_buf[e] = rew;
      }
    } else if (ztask_is<L, PULSE_ZTASK_REACH>(a)) {
      if constexpr (kServes<L, PULSE_ZTASK_REACH>) {
        const Vec3 tar = {a.tar_pos[3 * e], a.tar_pos[3 * e + 1], a.tar_pos[3 * e + 2]};
        const Vec3 lt = yaw_rot(yr, tar - p_root);  // compute_location_observations (humanoid_reach.py:224-236)
        t[0] = lt.x; t[1] = lt.y; t[2] = lt.z;
        if constexpr (kObsOnly) return;
        const Vec3 d = tar - p_reach;               // compute_reach_reward (:238-250)
        a.rew_buf[e] = expf(-4.0f * (d.x * d.x + d.y * d.y + d.z * d.z));
      }
    } else if constexpr (kServes<L, PULSE_ZTASK_STRIKE>) {
      const float* ts = a.target_states + e * a.target_env_stride;
      const Vec3 tp = {ts[0], ts[1], ts[2]};
      const Quat tq = {ts[3], ts[4], ts[5], ts[6]};
      // observation (:270-293): target position relative to the root with the ABSOLUTE height, 6D rotation, velocities, heading frame
      const Vec3 lp = yaw_rot(yr, Vec3{tp.x - p_root.x, tp.y - p_root.y, tp.z});
      t[0] = lp.x; t[1] = lp.y; t[2] = lp.z;
      qsix(yaw_mul_left(-hs, hc, tq), t + 3);
      const Vec3 lv = yaw_rot(yr, Vec3{ts[7], ts[8], ts[9]}), lw = yaw_rot(yr, Vec3{ts[10], ts[11], ts[12]});
      t[9] = lv.x; t[10] = lv.y; t[11] = lv.z;
      t[12] = lw.x; t[13] = lw.y; t[14] = lw.z;
      if constexpr (kObsOnly) return;
      // reward (:295-328)
      const float rot_err = 2.0f * tq.w * tq.w - 1.0f + 2.0f * tq.z * tq.z;      // z component of quat_rotate(tar_rot, [0, 0, 1])
      const float rot_r = fmaxf(1.0f - rot_err, 0.0f);
      float dx = tp.x - p_root.x, dy = tp.y - p_root.y;
      const float dn = fmaxf(sqrtf(dx * dx + dy * dy), 1e-12f);                    // torch.nn.functional.normalize (eps 1e-12)
      dx /= dn; dy /= dn;
      const float dir_speed = dx * vx + dy * vy;
      const float verr = fmaxf(1.0f - dir_speed, 0.0f);
      float vel_r = expf(-4.0f * verr * verr);
      if (dir_speed <= 0.0f) vel_r = 0.0f;
      float rew = 0.6f * rot_r + 0.4f * vel_r;
      if (rot_err < 0.2f) rew = 1.0f;
      a.rew_buf[e] = rew;
      // reset (:330-375): also fails when the target is pushed (> 50 N horizontally) while a non-strike body presses hard
      const float* tc = a.tar_contact_forces + e * a.tar_contact_env_stride;
      const bool tar_contact = fabsf(tc[0]) > 50.0f || fabsf(tc[1]) > 50.0f;
      failed = failed || (a.enable_early_termination && tar_contact && any_hard);
    }
    // fall_flags raises no flag without early termination, so for reach and speed the first term only restates `failed`
    const long long term = (a.enable_early_termination && failed && prog > 1) ? 1 : 0;
    a.terminate_buf[e] = term;
    a.reset_buf[e] = prog >= a.max_episode_length - 1 ? 1 : term;
  }
}

}  // namespace pulse
