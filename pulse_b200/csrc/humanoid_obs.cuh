// Humanoid observation layouts and per-env terms shared by the task step kernels (one warp per env, lane = body).
#pragma once
#include "pulse_common.cuh"
#include "quat_math.cuh"

namespace pulse {

namespace {  // __constant__ tables are per module; one copy in every translation unit that builds AMP rows
// kept joints (joint = body - 1), dropping L_Toe(3) R_Toe(7) L_Hand(17) R_Hand(22): humanoid.py:397,417-421
__constant__ int c_kept_joint[19] = {0, 1, 2, 4, 5, 6, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 19, 20, 21};
__constant__ int c_key_body[4] = {7, 3, 22, 17};  // R_Ankle, L_Ankle, R_Wrist, L_Wrist (env_im.yaml:36)
// SMPL-X: joints 0..50 without L_Toe(3) R_Toe(7) (humanoid.py:404-421, no hand joints dropped); key bodies R_Ankle, L_Ankle,
// R_Wrist, L_Wrist in SMPLH_MUJOCO_NAMES order (env_pulsex_amp.yaml key_bodies)
__constant__ int c_smplx_kept_joint[49] = {0,  1,  2,  4,  5,  6,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26,
                                           27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50};
__constant__ int c_smplx_key_body[4] = {7, 3, 36, 17};
}  // namespace

// The body layouts the latent-task step, reset and AMP code is instantiated for.  B bodies give a MotionLib frame record
// pos 3B | rot 4B | vel 3B | angvel 3B, an aux record lrs 4B | dvs 3(B - 1) | pad, and a self observation of 1 + 3(B - 1) + 6B + 3B + 3B
// floats.  kUpright: the step's self observation takes the heading of the root rotation itself (has_upright_start), otherwise
// of remove_base_rot(root).  kTasks: bit k set when the step serves task kind k (PULSE_ZTASK_*) through StepArgs.kind, or through
// the layout alone when it serves one kind; kPower: the speed task's power term.  The AMP observation
// (build_amp_observations_smpl with dof_subset) keeps kAmpJoints joints, kept_joint(i) for i < kAmpJoints, and the four key bodies
// key_body(i): kAmpObs = 1 + 6 + 3 + 3 + 9 kAmpJoints + 12 floats with the root height.
struct SmplLayout {
  static constexpr int kBodies = PULSE_NUM_BODIES, kDofs = PULSE_NUM_DOF, kSelfObs = PULSE_SELF_OBS;
  static constexpr int kFrameRec = PULSE_FRAME_REC, kAuxRec = PULSE_AUX_REC;
  static constexpr int kAmpJoints = 19, kAmpObs = PULSE_AMP_OBS;
  static constexpr bool kUpright = true, kPower = true;
  static constexpr unsigned kTasks = (1u << PULSE_ZTASK_SPEED) | (1u << PULSE_ZTASK_STRIKE);
  using StepArgs = pulse_ztask_step_args_t;
  __device__ static __forceinline__ int kept_joint(int i) { return c_kept_joint[i]; }
  __device__ static __forceinline__ int key_body(int i) { return c_key_body[i]; }
};
// The SMPL reach step: SmplLayout's geometry with the reach task's argument struct.
struct SmplReachLayout : SmplLayout {
  static constexpr bool kPower = false;
  static constexpr unsigned kTasks = 1u << PULSE_ZTASK_REACH;
  using StepArgs = pulse_reach_step_args_t;
};
struct SmplxLayout {
  static constexpr int kBodies = PULSE_SMPLX_BODIES, kDofs = PULSE_SMPLX_DOF, kSelfObs = PULSE_SMPLX_SELF_OBS;
  static constexpr int kFrameRec = PULSE_SMPLX_FRAME_REC, kAuxRec = PULSE_SMPLX_AUX_REC;
  static constexpr int kAmpJoints = 49, kAmpObs = PULSE_SMPLX_AMP_OBS;
  static constexpr bool kUpright = false, kPower = false;
  static constexpr unsigned kTasks = 1u << PULSE_ZTASK_SPEED;
  using StepArgs = pulse_smplx_speed_step_args_t;
  __device__ static __forceinline__ int kept_joint(int i) { return c_smplx_kept_joint[i]; }
  __device__ static __forceinline__ int key_body(int i) { return c_smplx_key_body[i]; }
};
// The SMPL-X reach and strike steps: SmplxLayout's geometry with their own argument struct.
struct SmplxTargetLayout : SmplxLayout {
  static constexpr unsigned kTasks = (1u << PULSE_ZTASK_REACH) | (1u << PULSE_ZTASK_STRIKE);
  using StepArgs = pulse_smplx_target_step_args_t;
};
static_assert(13 + 9 * SmplLayout::kAmpJoints + 12 == PULSE_AMP_OBS, "SMPL AMP observation");
static_assert(13 + 9 * SmplxLayout::kAmpJoints + 12 == PULSE_SMPLX_AMP_OBS, "SMPL-X AMP observation");
static_assert(PULSE_SMPLX_AMP_OBS - 1 == PULSE_SMPLX_AMP_OBS_NO_HEIGHT, "SMPL-X AMP observation without the root height");
static_assert(3 * PULSE_SMPLX_BODIES + 4 * PULSE_SMPLX_BODIES + 6 * PULSE_SMPLX_BODIES == PULSE_SMPLX_FRAME_REC, "SMPL-X frame record");
static_assert(4 * PULSE_SMPLX_BODIES + PULSE_SMPLX_DOF <= PULSE_SMPLX_AUX_REC && PULSE_SMPLX_AUX_REC % 4 == 0, "SMPL-X aux record");
static_assert(1 + 3 * (PULSE_SMPLX_BODIES - 1) + 12 * PULSE_SMPLX_BODIES == PULSE_SMPLX_SELF_OBS, "SMPL-X self observation");

// compute_humanoid_observations_smpl_max (humanoid.py:1675-1731) with local root obs and the root height: body j's slice of the
// self observation of B bodies [root height | (B-1) x position | B x six-D rotation | B x velocity | B x angular velocity] (358 floats
// for SMPL), all in the heading frame.  The heights p.z and p_root.z are taken from the task's reference (the ground, or the
// terrain's center height); (hs, hc) is the heading's half-angle sine / cosine and yr = make_yaw of the inverse heading.  The
// imitation step kernel writes the same layout inline (see im_step.cu).
template <int B = PULSE_NUM_BODIES>
__device__ __forceinline__ void store_self_obs(float* o, int j, Vec3 p, Vec3 p_root, Quat q, Vec3 v, Vec3 w, float hs, float hc, Yaw yr) {
  if (j == 0) o[0] = p_root.z;
  else stv(o + 1 + 3 * (j - 1), yaw_rot(yr, p - p_root));
  qsix(yaw_mul_left(-hs, hc, q), o + 3 * B - 2 + 6 * j);
  stv(o + 9 * B - 2 + 3 * j, yaw_rot(yr, v));
  stv(o + 12 * B - 2 + 3 * j, yaw_rot(yr, w));
}

struct AmpJoint {
  Vec3 exp_map;  // the joint's local rotation
  Vec3 vel;      // its three dof velocities
};

// build_amp_observations_smpl (humanoid_amp.py:924-969) with dof_to_obs_smpl (humanoid.py:1436-1446) in body layout L: one warp writes
// the L::kAmpObs-float AMP observation [h | six(hinv q0) | R v0 | R w0 | J x six(dof) | 3J dof velocities | 4 x R(key - p0)] of the
// root state (p0, q0, v0, w0), J = L::kAmpJoints (196 floats for SMPL, 466 for SMPL-X).  Lane 0 writes the root features, lane l the
// kept joints l, l + 32, ... below J, and the four lanes after the last joint lane of the last pass the key bodies (SMPL: joints on
// lanes 0..18, key bodies on 19..22; SMPL-X: joints on 0..31 and 0..16, key bodies on 17..20).  joint(jt) returns joint jt's AmpJoint,
// key_pos(kb) key body kb's world position.
template <class L = SmplLayout, class JointFn, class KeyPosFn>
__device__ __forceinline__ void store_amp_obs(float* o, int lane, Vec3 p0, Quat q0, Vec3 v0, Vec3 w0, JointFn joint, KeyPosFn key_pos) {
  constexpr int kJ = L::kAmpJoints, kPasses = (kJ + 31) / 32, kKey0 = kJ - 32 * (kPasses - 1);
  static_assert(kKey0 + 4 <= 32, "the key bodies share the last pass's warp");
  float hs, hc;
  heading_half(q0, hs, hc);
  const Quat h_inv = {0.0f, 0.0f, -hs, hc};
  const Yaw yr = make_yaw(h_inv);
  if (lane == 0) {
    o[0] = p0.z;
    qsix(qmul(h_inv, q0), o + 1);
    stv(o + 7, yaw_rot(yr, v0));
    stv(o + 10, yaw_rot(yr, w0));
  }
#pragma unroll 1
  for (int s = 0; s < kPasses; ++s) {   // not unrolled: two SMPL-X passes unrolled keep registers live across the sincos slow path
    const int i = lane + 32 * s;
    if (i < kJ) {
      const AmpJoint jt = joint(L::kept_joint(i));
      qsix(exp_map_quat(jt.exp_map), o + 13 + 6 * i);
      stv(o + 13 + 6 * kJ + 3 * i, jt.vel);
    } else if (s == kPasses - 1 && lane < kKey0 + 4) {
      stv(o + 13 + 9 * kJ + 3 * (lane - kKey0), yaw_rot(yr, key_pos(L::key_body(lane - kKey0)) - p0));
    }
  }
}

// store_amp_obs from the simulator state of env e: the root and key bodies from body_state ([pos | quat | vel | ang vel] per body),
// the joints from the dof position / velocity views.
template <class L = SmplLayout, class Args>
__device__ __forceinline__ void store_amp_obs_sim(float* o, int lane, const Args& a, long long e) {
  const float* bs = a.body_state + e * a.body_env_stride;
  const float* dp = a.dof_pos + e * a.dof_env_stride;
  const float* dv = a.dof_vel + e * a.dof_env_stride;
  const long long ds = a.dof_elem_stride;
  const auto joint = [&](int jt) {
    return AmpJoint{{dp[(3 * jt + 0) * ds], dp[(3 * jt + 1) * ds], dp[(3 * jt + 2) * ds]},
                    {dv[(3 * jt + 0) * ds], dv[(3 * jt + 1) * ds], dv[(3 * jt + 2) * ds]}};
  };
  const auto key_pos = [&](int kb) { return ldv(bs + kb * PULSE_BODY_STATE_W); };
  store_amp_obs<L>(o, lane, ldv(bs), ldq(bs + 3), ldv(bs + 7), ldv(bs + 10), joint, key_pos);
}

// The fall test of compute_humanoid_reset (humanoid.py:1573-1608) for body lane j of env e: `contact` when a body that may not
// touch the ground has a contact force component above 0.1 N, `height` when such a body is below its termination height.  The env
// has fallen when some lane has `contact` and some lane has `height`.
struct FallFlags {
  bool contact, height;
};
template <class Args>
__device__ __forceinline__ FallFlags fall_flags(const Args& a, long long e, int j, bool body, float z) {
  FallFlags f = {false, false};
  if (a.enable_early_termination && body && !((a.contact_body_mask >> j) & 1u)) {   // a 32- or 64-bit mask
    if (a.contact_forces != nullptr) {
      const float* cf = a.contact_forces + e * a.contact_env_stride + j * 3;
      f.contact = fabsf(cf[0]) > 0.1f || fabsf(cf[1]) > 0.1f || fabsf(cf[2]) > 0.1f;
    }
    f.height = z < a.termination_heights[j];
  }
  return f;
}

// sum |tau * qdot| over the 69 dofs of env e, in every lane: the power term (humanoid_speed.py:215-222)
template <class Args>
__device__ __forceinline__ float dof_power(const Args& a, long long e, int lane) {
  const float* fr = a.dof_force + e * a.dof_force_stride;
  const float* dv = a.dof_vel + e * a.dof_env_stride;
  float power = 0.0f;
  for (int d = lane; d < PULSE_NUM_DOF; d += 32) power += fabsf(fr[d] * dv[d * a.dof_elem_stride]);
  return warp_sum(power);
}

}  // namespace pulse
