// HumanoidPedestrianTerrain(Z) (phc/env/tasks/humanoid_pedestrian_terrain.py) on the device:
//   terrain_step_kernel   reward, reset and observation of post_physics_step in one launch, one warp per env (lane = body):
//                         _compute_reward :871-896, _compute_reset :849-869 -> compute_humanoid_reset :1477-1531,
//                         _compute_humanoid_obs :195-223, _compute_task_obs :385-440 (compute_location_observations :1588-1616,
//                         get_heights :718-772 at the head pose :296-311, get_center_heights :690-716).
//   terrain_rollout_kernel  the same per-env code (terrain_env) for the rollout: progress_buf += 1 first, dones afterwards.
//   traj_reset_kernel     TrajGenerator.reset (phc/utils/traj_generator.py:57-112), one thread per reset env;
//   traj_list_kernel      the same over the device-side env list of a reset (pulse_traj_reset_list).
//   terrain_heights_kernel get_center_heights / get_heights alone (the spawn lift of _reset_ref_state_init :527-584).
// Height sampling (terrain_height.cuh) is Terrain.world_points_to_map / sample_height_points (:1191-1198, :1261-1267); trajectory lookups are
// TrajGenerator.calc_pos (traj_generator.py:148-165).
//
// Cell indices, the reset mask and the trajectory segment indices are integers decided by fp32 arithmetic, so the operations that
// feed them keep the reference's order with round-to-nearest intrinsics (no FMA contraction), as in im_step.cu.  Everything else
// is under the 1e-4 float tolerance of the observations and rewards.
#include "philox.cuh"
#include "terrain_height.cuh"

namespace pulse {
namespace {

constexpr int kTB = PULSE_NUM_BODIES;
constexpr int kVerts = PULSE_TRAJ_VERTS;
constexpr unsigned long long kTrajListStream = 4ull << 32;   // Philox index e + 4 * 2^32: pulse_traj_reset_list

// calc_heading_quat / calc_heading_quat_inv (phc/utils/torch_utils.py:200-240) in the angle form the reference computes: heading =
// atan2 of the rotated x axis, quat_from_angle_axis(+-heading, z) incl. its final quat_unit.  The height-map points rotate by it, so
// their cell indices follow it; heading_half() would move them by ~2e-7.
__device__ __forceinline__ Quat heading_quat_ref(Quat q, bool inverse) {
  const float s = __fsub_rn(__fmul_rn(2.0f, __fmul_rn(q.w, q.w)), 1.0f);
  const float rx = __fadd_rn(s, __fmul_rn(__fmul_rn(q.x, q.x), 2.0f));
  const float ry = __fadd_rn(__fmul_rn(__fmul_rn(q.z, q.w), 2.0f), __fmul_rn(__fmul_rn(q.y, q.x), 2.0f));
  float h = atan2f(ry, rx);
  if (inverse) h = -h;
  float sn, cs;
  sincosf(__fmul_rn(h, 0.5f), &sn, &cs);
  const float n = fmaxf(__fsqrt_rn(__fadd_rn(__fmul_rn(sn, sn), __fmul_rn(cs, cs))), 1e-9f);
  return {0.0f, 0.0f, __fdiv_rn(sn, n), __fdiv_rn(cs, n)};
}

// TrajGenerator.calc_pos (traj_generator.py:148-165): phase = clip(t / (num_verts * dt), 0, 1) -- num_verts, not num_segs, as in the
// reference -- then the floor / ceil waypoints and their lerp, each operation rounded as the reference rounds it.
__device__ __forceinline__ Vec3 traj_pos(const float* verts, float t, float traj_dur) {
  const float phase = fminf(fmaxf(__fdiv_rn(t, traj_dur), 0.0f), 1.0f);
  const float seg = __fmul_rn(phase, static_cast<float>(kVerts - 1));
  const int i0 = static_cast<int>(floorf(seg)), i1 = static_cast<int>(ceilf(seg));
  const float b = __fsub_rn(seg, static_cast<float>(i0));
  const float* p0 = verts + 3 * i0;
  const float* p1 = verts + 3 * i1;
  return {lerp_rn(p0[0], p1[0], b), lerp_rn(p0[1], p1[1], b), lerp_rn(p0[2], p1[2], b)};
}

// The per-env work of both step kernels: reward, reset and observation of env e as a.flags selects them, one warp (lane = body).
// `prog` is progress_buf[e] as every lane of the warp must see it; the body does not read the counter itself.
__device__ __forceinline__ void terrain_env(const pulse_terrain_step_args_t& a, const HeightField& hfield, long long e, long long prog, int lane) {
  const bool upright = a.upright != 0;
  const int j = lane;
  const bool body = j < kTB;
  const float* bs = a.body_state + e * a.body_env_stride + (body ? j : 0) * 13;
  const Vec3 p = {bs[0], bs[1], bs[2]};
  const Vec3 p_root = {__shfl_sync(kFull, p.x, 0), __shfl_sync(kFull, p.y, 0), __shfl_sync(kFull, p.z, 0)};
  const float* rs = a.root_states + e * a.root_env_stride;
  const Vec3 a_pos = {rs[0], rs[1], rs[2]};
  const float t_now = __fmul_rn(__ll2float_rn(prog), a.dt);   // progress_buf * dt
  const float* verts = a.traj_verts + e * (kVerts * 3);

  if (a.flags & PULSE_STEP_REWARD) {
    // _compute_reward (:871-896): location reward against the ACTOR root state; the power term is always reported in reward_raw[:, 1]
    const float power = a.dof_force != nullptr ? -a.power_coefficient * dof_power(a, e, lane) : 0.0f;
    if (lane == 0) {
      const Vec3 tar = traj_pos(verts, t_now, a.traj_dur);
      const float dx = tar.x - a_pos.x, dy = tar.y - a_pos.y;
      float err = dx * dx + dy * dy;
      if (a.fuzzy_target && err < 0.0025f) err = 0.0f;   // compute_location_reward_fuzzy (:1633-1646)
      const float loc = expf(-2.0f * err);                // compute_location_reward (:1620-1630)
      a.rew_buf[e] = a.power_reward ? loc + power : loc;
      if (a.reward_raw != nullptr) {
        a.reward_raw[e * a.raw_stride] = loc;
        a.reward_raw[e * a.raw_stride + 1] = power;
      }
    }
  }

  if (a.flags & PULSE_STEP_RESET) {
    // compute_humanoid_reset (:1477-1531): the contact force summed over the non-contact bodies, in body order, has norm > 50
    // (after progress 1), or the RIGID-BODY root is more than fail_dist from the trajectory point.  center_height and the
    // termination heights are unused by the reference.
    Vec3 f = {0.0f, 0.0f, 0.0f};
    if (a.enable_early_termination && body && !((a.contact_body_mask >> j) & 1u)) {
      const float* cf = a.contact_forces + e * a.contact_env_stride + j * 3;
      f = {cf[0], cf[1], cf[2]};
    }
    Vec3 s = {0.0f, 0.0f, 0.0f};
    for (int b = 0; b < kTB; ++b) {
      s.x = __fadd_rn(s.x, __shfl_sync(kFull, f.x, b));
      s.y = __fadd_rn(s.y, __shfl_sync(kFull, f.y, b));
      s.z = __fadd_rn(s.z, __shfl_sync(kFull, f.z, b));
    }
    if (lane == 0) {
      long long term = 0;
      if (a.enable_early_termination) {
        const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(s.x, s.x), __fmul_rn(s.y, s.y)), __fmul_rn(s.z, s.z)));
        const bool fallen = nrm > 50.0f && prog > 1;
        const Vec3 tar = traj_pos(verts, t_now, a.traj_dur);
        const float dx = __fsub_rn(tar.x, p_root.x), dy = __fsub_rn(tar.y, p_root.y);
        const bool far = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) > __fmul_rn(a.fail_dist, a.fail_dist);
        term = (!a.no_collision_check && (fallen || far)) ? 1 : 0;
      }
      a.terminate_buf[e] = term;
      a.reset_buf[e] = prog >= a.max_episode_length - 1 ? 1 : term;
    }
  }

  if (a.flags & PULSE_STEP_OBS) {
    const Quat q = {bs[3], bs[4], bs[5], bs[6]};
    const Vec3 v = {bs[7], bs[8], bs[9]}, w = {bs[10], bs[11], bs[12]};
    const Quat q_root = {__shfl_sync(kFull, q.x, 0), __shfl_sync(kFull, q.y, 0), __shfl_sync(kFull, q.z, 0), __shfl_sync(kFull, q.w, 0)};
    float* o = a.obs_buf + e * a.obs_stride;
    // _compute_humanoid_obs (:195-223): every body's z minus the mean center height around the rigid-body root, then
    // compute_humanoid_observations_smpl_max (humanoid.py:1675-1731) with local root obs and the root height
    const float c_self = center_height(hfield, a.center_points, a.num_center_points, q_root, p_root, upright, lane);
    float hs, hc;
    heading_half(base_rot_removed(q_root, upright), hs, hc);
    const Yaw yr = make_yaw(Quat{0.0f, 0.0f, -hs, hc});
    // _compute_task_obs (:385-440).  Trajectory samples at progress * dt + k * trajSampleTimestep (humanoid_traj.py:196-211) in the
    // heading frame of the actor root (compute_location_observations :1588-1616), xy only.
    const Quat a_rot = {rs[3], rs[4], rs[5], rs[6]};
    float* t = o + PULSE_SELF_OBS;
    if (lane < a.num_traj_samples) {
      const float tk = __fadd_rn(t_now, __fmul_rn(static_cast<float>(lane), a.traj_sample_timestep));
      const Vec3 tp = traj_pos(verts, tk, a.traj_dur);
      const Vec3 d = qrot(heading_quat_ref(base_rot_removed(a_rot, upright), true), tp - a_pos);
      t[2 * lane] = d.x;
      t[2 * lane + 1] = d.y;
    }
    // the self observation is stored after the trajectory samples: in the other order ptxas spills a register
    const Vec3 pc = {p.x, p.y, p.z - c_self}, rc = {p_root.x, p_root.y, p_root.z - c_self};
    if (body) store_self_obs(o, j, pc, rc, q, v, w, hs, hc, yr);
    // height map at the head pose (get_head_pose :296-311, get_heights :718-772), relative to the mean center height around the
    // actor root (use_center_height) or to the actor root's z, clipped to +-3 m and scaled by 5
    const float ref_h = a.use_center_height ? center_height(hfield, a.center_points, a.num_center_points, a_rot, a_pos, upright, lane)
                                            : a_pos.z;
    const Vec3 head_p = {__shfl_sync(kFull, p.x, a.head_body_id), __shfl_sync(kFull, p.y, a.head_body_id),
                         __shfl_sync(kFull, p.z, a.head_body_id)};
    const Quat head_q = {__shfl_sync(kFull, q.x, a.head_body_id), __shfl_sync(kFull, q.y, a.head_body_id),
                         __shfl_sync(kFull, q.z, a.head_body_id), __shfl_sync(kFull, q.w, a.head_body_id)};
    const Quat hq = heading_quat_ref(base_rot_removed(head_q, upright), false);
    float* hobs = t + 2 * a.num_traj_samples;
    for (int i = lane; i < a.num_height_points; i += 32) {
      const float m = height_at(hfield, hq, a.height_points + 3 * i, head_p);
      hobs[i] = fminf(fmaxf(ref_h - m, -3.0f), 3.0f) * 5.0f;
    }
  }
}

__global__ void __launch_bounds__(256) terrain_step_kernel(const pulse_terrain_step_args_t a, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const HeightField hfield = {a.heightfield, a.hf_rows, a.hf_cols, a.horizontal_scale, a.vertical_scale};
  long long rows = n;
  if (a.env_ids != nullptr && a.env_count != nullptr) rows = min(rows, static_cast<long long>(*a.env_count));
  for (long long r = blockIdx.x * 8ll + warp; r < rows; r += 8ll * gridDim.x) {
    const long long e = a.env_ids != nullptr ? a.env_ids[r] : r;
    terrain_env(a, hfield, e, a.progress_buf[e], lane);
  }
}

// pulse_terrain_rollout_step: lane 0 advances progress_buf[e] (humanoid.py:1317) and broadcasts the new value to the warp, so no
// lane reads the counter from memory; then every step of PULSE_STEP_ALL, then dones[e] = float(reset_buf[e]) (amp_agent.py:380).
__global__ void __launch_bounds__(256) terrain_rollout_kernel(const pulse_terrain_step_args_t a, float* __restrict__ dones, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const HeightField hfield = {a.heightfield, a.hf_rows, a.hf_cols, a.horizontal_scale, a.vertical_scale};
  long long* progress = const_cast<long long*>(reinterpret_cast<const long long*>(a.progress_buf));
  for (long long e = blockIdx.x * 8ll + warp; e < n; e += 8ll * gridDim.x) {
    long long prog = 0;
    if (lane == 0) {
      prog = progress[e] + 1;
      progress[e] = prog;
    }
    prog = __shfl_sync(kFull, prog, 0);
    terrain_env(a, hfield, e, prog, lane);
    if (lane == 0) dones[e] = static_cast<float>(a.reset_buf[e]);
  }
}

// TrajGenerator.reset (traj_generator.py:57-112) for one env.  Injected draws per env (PULSE_TRAJ_DRAWS = 4 * S + 2, S = num_verts - 1):
// [0, S) turn angles, [S, 2S) sharp-turn angles, [2S, 3S) sharp-turn coins (sharp where u < sharp_turn_prob, the bernoulli draw),
// [3S, 4S) speed changes, 4S initial heading, 4S + 1 initial speed.  Column 0 of the first four rows is overwritten, as in the
// reference.  Without injected draws, Philox block (seed, index, ctr0 + k) supplies the four draws of segment k and block
// (seed, index, ctr0 + S) the initial heading and speed: a different stream from torch's generator, the same distribution.
// torch.cumsum on the CPU accumulates fp32 in double; so do the two running sums here.  Args is pulse_traj_reset_args_t or
// pulse_traj_list_args_t (the same trajectory parameters).
template <class Args>
__device__ __forceinline__ void traj_generate(const Args& a, float* vt, float x0, float y0, const float* rin, unsigned long long index,
                                              unsigned long long ctr0) {
  constexpr int S = kVerts - 1;
  float u_head, u_v0;
  if (rin != nullptr) {
    u_head = rin[4 * S];
    u_v0 = rin[4 * S + 1];
  } else {
    const Philox4 b = philox4x32_10(a.seed, index, ctr0 + S);
    u_head = u01(b.x);
    u_v0 = u01(b.y);
  }
  const float pi = 3.14159265358979f;
  vt[0] = x0;
  vt[1] = y0;
  double ang = 0.0, px = 0.0, py = 0.0;
  float speed = 0.0f;
  for (int k = 0; k < S; ++k) {
    float u_turn, u_sharp, coin, u_speed;
    if (rin != nullptr) {
      u_turn = rin[k];
      u_sharp = rin[S + k];
      coin = rin[2 * S + k];
      u_speed = rin[3 * S + k];
    } else {
      const Philox4 b = philox4x32_10(a.seed, index, ctr0 + k);
      u_turn = u01(b.x);
      u_sharp = u01(b.y);
      coin = u01(b.z);
      u_speed = u01(b.w);
    }
    float dth;
    if (k == 0) dth = __fmul_rn(pi, __fsub_rn(__fmul_rn(2.0f, u_head), 1.0f));
    else if (coin < a.sharp_turn_prob) dth = __fmul_rn(pi, __fsub_rn(__fmul_rn(2.0f, u_sharp), 1.0f));
    else dth = __fmul_rn(__fsub_rn(__fmul_rn(2.0f, u_turn), 1.0f), a.dtheta_scale);
    if (k == 0) speed = __fadd_rn(__fmul_rn(__fsub_rn(a.speed_max, a.speed_min), u_v0), a.speed_min);
    else speed = fminf(fmaxf(__fadd_rn(speed, __fmul_rn(__fsub_rn(__fmul_rn(2.0f, u_speed), 1.0f), a.dspeed_scale)), a.speed_min), a.speed_max);
    ang += static_cast<double>(dth);
    const float th = static_cast<float>(ang);
    float sn, cs;
    sincosf(th, &sn, &cs);
    const float seg = __fmul_rn(speed, a.seg_dt);
    float dx = __fmul_rn(cs, seg), dy = __fmul_rn(-sn, seg);
    if (k == 0) {
      dx = __fadd_rn(dx, x0);
      dy = __fadd_rn(dy, y0);
    }
    px += static_cast<double>(dx);
    py += static_cast<double>(dy);
    vt[3 * (k + 1)] = static_cast<float>(px);
    vt[3 * (k + 1) + 1] = static_cast<float>(py);
    vt[3 * (k + 1) + 2] = 0.0f;
  }
}

// pulse_traj_reset: row i of the id list; Philox keyed (seed, env, offset + *offset_dev + k).
__global__ void __launch_bounds__(128) traj_reset_kernel(const pulse_traj_reset_args_t a) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= a.num_ids) return;
  const long long e = a.env_ids[i];
  const unsigned long long off = a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull);
  traj_generate(a, a.verts + e * (kVerts * 3), a.init_pos[i * a.init_stride], a.init_pos[i * a.init_stride + 1],
                a.rand != nullptr ? a.rand + i * PULSE_TRAJ_DRAWS : nullptr, static_cast<unsigned long long>(e), off);
}

// pulse_traj_reset_list: the envs of a device-side list, starting at root_states[e, 0:2]; draws per ENV, or Philox keyed
// (seed, e + 4 * 2^32, PULSE_TRAJ_VERTS * (offset + *offset_dev) + k), so resets at different offsets never share a block.
__global__ void __launch_bounds__(128) traj_list_kernel(const pulse_traj_list_args_t a) {
  const long long n = *a.count;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = a.env_list[i];
    const unsigned long long off = a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull);
    const float* rs = a.root_states + e * a.root_env_stride;
    traj_generate(a, a.verts + e * (kVerts * 3), rs[0], rs[1], a.rand != nullptr ? a.rand + e * PULSE_TRAJ_DRAWS : nullptr,
                  static_cast<unsigned long long>(e) + kTrajListStream, static_cast<unsigned long long>(kVerts) * off);
  }
}

__global__ void __launch_bounds__(256) terrain_heights_kernel(const pulse_terrain_heights_args_t a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const HeightField hfield = {a.heightfield, a.hf_rows, a.hf_cols, a.horizontal_scale, a.vertical_scale};
  for (long long r = blockIdx.x * 8ll + warp; r < a.num_rows; r += 8ll * gridDim.x) {
    const float* rs = a.root_states + r * a.root_stride;
    const Vec3 org = {rs[0], rs[1], rs[2]};
    Quat q = base_rot_removed(Quat{rs[3], rs[4], rs[5], rs[6]}, a.upright != 0);
    q = a.mode == PULSE_HEIGHTS_CENTER ? yaw_only(q) : heading_quat_ref(q, false);
    for (int i = lane; i < a.num_points; i += 32) a.heights[r * a.heights_stride + i] = height_at(hfield, q, a.points + 3 * i, org);
  }
}

int check_heightfield(const char* who, const int16_t* hf, int64_t rows, int64_t cols, float hscale) {
  PULSE_REQUIRE(hf == nullptr || (rows >= 2 && cols >= 2), "%s: heightfield needs at least 2 x 2 cells", who);
  PULSE_REQUIRE(hf == nullptr || hscale > 0.0f, "%s: horizontal_scale must be positive", who);
  return PULSE_OK;
}

// The argument checks of pulse_terrain_step, shared with pulse_terrain_rollout_step (`who` names the entry point).
int check_step_args(const char* who, const pulse_terrain_step_args_t& a, int64_t num_envs) {
  PULSE_REQUIRE(num_envs > 0, "%s: num_envs must be positive", who);
  PULSE_REQUIRE((a.flags & ~PULSE_STEP_ALL) == 0 && a.flags != 0, "%s: flags must be a non-empty set of REWARD / RESET / OBS", who);
  PULSE_REQUIRE(a.body_state && a.root_states && a.progress_buf && a.traj_verts, "%s: null input buffer", who);
  PULSE_REQUIRE(a.body_env_stride >= 24 * 13 && a.root_env_stride >= 13, "%s: body / root strides too small", who);
  PULSE_REQUIRE(a.dt > 0.0f && a.traj_dur > 0.0f, "%s: dt and traj_dur must be positive", who);
  PULSE_REQUIRE(a.env_ids == nullptr || a.flags == PULSE_STEP_OBS, "%s: env_ids only with PULSE_STEP_OBS", who);
  if (a.flags & PULSE_STEP_REWARD) {
    PULSE_REQUIRE(a.rew_buf != nullptr, "%s: reward needs rew_buf", who);
    PULSE_REQUIRE(!(a.power_reward || a.reward_raw) || (a.dof_force && a.dof_vel && a.dof_elem_stride >= 1),
                  "%s: the power term (power_reward / reward_raw) needs dof_force and dof_vel", who);
    PULSE_REQUIRE(a.reward_raw == nullptr || a.raw_stride >= 2, "%s: raw_stride < 2", who);
  }
  if (a.flags & PULSE_STEP_RESET) {
    PULSE_REQUIRE(a.reset_buf && a.terminate_buf, "%s: reset needs reset_buf and terminate_buf", who);
    PULSE_REQUIRE(!a.enable_early_termination || (a.contact_forces && a.contact_env_stride >= 24 * 3),
                  "%s: early termination needs contact_forces with env stride >= 72", who);
  }
  if (a.flags & PULSE_STEP_OBS) {
    PULSE_REQUIRE(a.obs_buf && a.height_points && a.center_points, "%s: observation needs obs_buf, height_points, center_points", who);
    PULSE_REQUIRE(a.num_traj_samples >= 1 && a.num_traj_samples <= 32, "%s: num_traj_samples %d not in [1, 32]", who, a.num_traj_samples);
    PULSE_REQUIRE(a.num_height_points >= 1 && a.num_center_points >= 1, "%s: empty point set", who);
    PULSE_REQUIRE(a.head_body_id >= 0 && a.head_body_id < 24, "%s: head_body_id %d out of range", who, a.head_body_id);
    PULSE_REQUIRE(a.obs_stride >= PULSE_SELF_OBS + 2 * a.num_traj_samples + a.num_height_points, "%s: obs_stride %lld too small", who,
                  (long long)a.obs_stride);
    return check_heightfield(who, a.heightfield, a.hf_rows, a.hf_cols, a.horizontal_scale);
  }
  return PULSE_OK;
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_terrain_step(const pulse_terrain_step_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_terrain_step: null args");
  const pulse_terrain_step_args_t& a = *args;
  const int st = check_step_args("pulse_terrain_step", a, num_envs);
  if (st != PULSE_OK) return st;
  terrain_step_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("terrain_step_kernel");
  return PULSE_OK;
}

extern "C" int pulse_terrain_rollout_step(const pulse_terrain_step_args_t* args, float* dones, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args && dones, "pulse_terrain_rollout_step: null args / dones");
  const pulse_terrain_step_args_t& a = *args;
  PULSE_REQUIRE(a.flags == PULSE_STEP_ALL, "pulse_terrain_rollout_step: flags must be PULSE_STEP_ALL (reward, reset and observation)");
  const int st = check_step_args("pulse_terrain_rollout_step", a, num_envs);
  if (st != PULSE_OK) return st;
  terrain_rollout_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, dones, (long long)num_envs);
  PULSE_LAUNCH_OK("terrain_rollout_kernel");
  return PULSE_OK;
}

extern "C" int pulse_traj_reset(const pulse_traj_reset_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_traj_reset: null args");
  const pulse_traj_reset_args_t& a = *args;
  PULSE_REQUIRE(a.num_ids >= 0, "pulse_traj_reset: negative num_ids");
  if (a.num_ids == 0) return PULSE_OK;
  PULSE_REQUIRE(a.env_ids && a.init_pos && a.verts, "pulse_traj_reset: null buffer");
  PULSE_REQUIRE(a.init_stride >= 2, "pulse_traj_reset: init_stride < 2");
  PULSE_REQUIRE(a.seg_dt > 0.0f && a.speed_max >= a.speed_min, "pulse_traj_reset: bad trajectory parameters");
  const long long blocks = (a.num_ids + 127) / 128;
  traj_reset_kernel<<<static_cast<unsigned>(blocks), 128, 0, static_cast<cudaStream_t>(stream)>>>(a);
  PULSE_LAUNCH_OK("traj_reset_kernel");
  return PULSE_OK;
}

extern "C" int pulse_terrain_heights(const pulse_terrain_heights_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_terrain_heights: null args");
  const pulse_terrain_heights_args_t& a = *args;
  PULSE_REQUIRE(a.mode == PULSE_HEIGHTS_CENTER || a.mode == PULSE_HEIGHTS_GRID, "pulse_terrain_heights: unknown mode %d", a.mode);
  PULSE_REQUIRE(a.num_rows >= 0 && a.num_points >= 1, "pulse_terrain_heights: bad sizes");
  if (a.num_rows == 0) return PULSE_OK;
  PULSE_REQUIRE(a.root_states && a.points && a.heights, "pulse_terrain_heights: null buffer");
  PULSE_REQUIRE(a.root_stride >= 7 && a.heights_stride >= a.num_points, "pulse_terrain_heights: strides too small");
  const int st = check_heightfield("pulse_terrain_heights", a.heightfield, a.hf_rows, a.hf_cols, a.horizontal_scale);
  if (st != PULSE_OK) return st;
  terrain_heights_kernel<<<grid_for(a.num_rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  PULSE_LAUNCH_OK("terrain_heights_kernel");
  return PULSE_OK;
}

extern "C" int pulse_traj_reset_list(const pulse_traj_list_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_traj_reset_list: null args");
  const pulse_traj_list_args_t& a = *args;
  PULSE_REQUIRE(num_envs >= 0 && num_envs < (1ll << 31), "pulse_traj_reset_list: num_envs %lld outside [0, 2^31)", (long long)num_envs);
  PULSE_REQUIRE(a.env_list && a.count && a.root_states && a.verts, "pulse_traj_reset_list: null list / count / root_states / verts");
  PULSE_REQUIRE(a.root_env_stride >= 2, "pulse_traj_reset_list: root_env_stride < 2");
  PULSE_REQUIRE(a.seg_dt > 0.0f && a.speed_max >= a.speed_min, "pulse_traj_reset_list: bad trajectory parameters");
  if (num_envs == 0) return PULSE_OK;
  traj_list_kernel<<<grid_for(num_envs, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(a);
  PULSE_LAUNCH_OK("traj_list_kernel");
  return PULSE_OK;
}
