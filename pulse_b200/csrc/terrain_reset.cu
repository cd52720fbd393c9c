// Reference-state reset of the pedestrian terrain task on the device, no host synchronisation (pulse_reset_terrain).  Two launches:
//   reset_compact_kernel  (reset_warps.cuh) the ordered compaction of the reset mask or id list into the env / actor lists and a count;
//   terrain_reset_kernel  one warp per (reset env, AMP history step k): the shared reset_warps work (clip, start time, MotionLib gather,
//                         SMPL ground fix, _set_env_state, counters, AMP rows) with the spawn of _reset_ref_state_init
//                         (humanoid_pedestrian_terrain.py:527-589) in place of a pose adjustment.
// The observation of the reset envs (pulse_terrain_step over the list) and the waypoints (pulse_traj_reset_list) follow.  Entry point,
// argument structs and Philox word layout: include/pulse_b200.h.
#include "reset_warps.cuh"
#include "terrain_height.cuh"

namespace pulse {
namespace {

__global__ void __launch_bounds__(kResetWarps * 32) terrain_reset_kernel(const pulse_motionlib_desc_t lib, const pulse_ztask_reset_args_t a,
                                                                          const pulse_terrain_spawn_args_t s) {
  __shared__ float stage_all[kResetWarps][PULSE_AMP_OBS];
  const bool upright = a.upright != 0;
  const HeightField hfield = {s.heightfield, s.hf_rows, s.hf_cols, s.horizontal_scale, s.vertical_scale};
  const auto spawn = [&](long long e, int lane, const Philox4& r0, unsigned long long, Vec3& p, Quat&, Vec3&, Vec3& rp, Quat& rr, Vec3&,
                         Vec3&) {
    // sample_valid_locations (:1175-1189): coord_{x,y}_scale[randint(0, num_samples)]
    long long l = s.loc_ids_in != nullptr ? s.loc_ids_in[e]
                                          : static_cast<long long>((static_cast<unsigned long long>(r0.z) * static_cast<unsigned long long>(s.num_locations)) >> 32);
    l = l < 0 ? 0 : (l >= s.num_locations ? s.num_locations - 1 : l);
    if (lane == 0 && s.loc_ids_out != nullptr) s.loc_ids_out[e] = l;
    const float nx = s.coord_x[l], ny = s.coord_y[l];
    const float dx = __fsub_rn(nx, rp.x), dy = __fsub_rn(ny, rp.y);   // diff_xy = new_root_xy - root_pos[:, 0:2]
    rp.x = nx;
    rp.y = ny;
    // root_pos[:, 2] += get_center_heights(cat[root_pos, root_rot]).mean(-1) (:556-563)
    rp.z = __fadd_rn(rp.z, center_height(hfield, s.center_points, static_cast<int>(s.num_center_points), rr, rp, upright, lane));
    // rb_pos[..., 0:2] += diff_xy (:566); the bodies' z is not lifted (the lift goes to key_pos, which is not read again)
    p.x = __fadd_rn(p.x, dx);
    p.y = __fadd_rn(p.y, dy);
  };
  reset_warps<SmplLayout>(lib, a, s.loc_ids_in == nullptr, stage_all[threadIdx.x >> 5], spawn);
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_reset_terrain(const pulse_motionlib_t* lib, const pulse_ztask_reset_args_t* args, const pulse_terrain_spawn_args_t* spawn,
                                   int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && args != nullptr && spawn != nullptr, "pulse_reset_terrain: null lib/args/spawn");
  const pulse_ztask_reset_args_t& a = *args;
  const pulse_terrain_spawn_args_t& s = *spawn;
  PULSE_REQUIRE(num_envs >= 0 && num_envs < (1ll << 31), "pulse_reset_terrain: num_envs %lld outside [0, 2^31)", (long long)num_envs);
  PULSE_REQUIRE(a.reset_buf != nullptr || a.env_ids_in != nullptr, "pulse_reset_terrain: neither a reset mask nor an env id list");
  PULSE_REQUIRE(a.env_ids_in == nullptr || (a.num_ids >= 0 && a.num_ids <= num_envs), "pulse_reset_terrain: num_ids %lld outside [0, %lld]",
                (long long)a.num_ids, (long long)num_envs);
  PULSE_REQUIRE(a.env_list != nullptr && a.count != nullptr, "pulse_reset_terrain: env_list / count outputs are required");
  PULSE_REQUIRE(a.sampled_motion_ids && a.motion_start_times && a.progress_buf, "pulse_reset_terrain: null task buffer");
  PULSE_REQUIRE(a.root_states && a.dof_pos && a.dof_vel && a.rigid_body_state, "pulse_reset_terrain: null simulator tensor");
  PULSE_REQUIRE(a.root_env_stride >= PULSE_BODY_STATE_W && a.dof_elem_stride >= 1 && a.dof_env_stride >= PULSE_NUM_DOF * a.dof_elem_stride &&
                a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "pulse_reset_terrain: bad root / dof / rigid-body strides");
  PULSE_REQUIRE(a.contact_forces == nullptr || (a.contact_bodies >= 0 && a.contact_env_stride >= 3 * a.contact_bodies),
                "pulse_reset_terrain: bad contact-force strides");
  PULSE_REQUIRE(a.target_states == nullptr, "pulse_reset_terrain: the terrain task has no target actor (target_states must be NULL)");
  PULSE_REQUIRE(a.floor != nullptr && a.floor_len >= lib->d.total_frames, "pulse_reset_terrain: floor table of %lld frames, the MotionLib has %lld",
                (long long)a.floor_len, (long long)lib->d.total_frames);
  PULSE_REQUIRE(a.motion_ids_in != nullptr || (a.sampling_cdf != nullptr && lib->d.num_motions >= 1),
                "pulse_reset_terrain: null sampling_cdf (needed to draw the clips)");
  PULSE_REQUIRE(a.pose_mode == PULSE_ZPOSE_AS_IS, "pulse_reset_terrain: pose_mode %d, the terrain task places the root itself (AS_IS)", a.pose_mode);
  PULSE_REQUIRE(a.state_init == PULSE_ZINIT_RANDOM, "pulse_reset_terrain: state_init %d, the terrain task always samples the start time (RANDOM)",
                a.state_init);
  PULSE_REQUIRE(a.amp_obs_buf == nullptr || (a.num_amp_steps >= 1 && a.num_amp_steps <= 16), "pulse_reset_terrain: num_amp_steps outside [1,16]");
  PULSE_REQUIRE(a.amp_fresh == nullptr || a.amp_obs_buf != nullptr, "pulse_reset_terrain: amp_fresh flags need the back-filled amp_obs_buf");
  PULSE_REQUIRE(a.amp_obs_buf == nullptr || a.amp_width == PULSE_AMP_OBS || a.amp_width == PULSE_AMP_OBS_NO_HEIGHT,
                "pulse_reset_terrain: amp_width %d is neither %d nor %d", a.amp_width, PULSE_AMP_OBS, PULSE_AMP_OBS_NO_HEIGHT);
  PULSE_REQUIRE(lib->d.aux_rec != nullptr, "pulse_reset_terrain: the MotionLib handle has no aux records (dof_pos / dof_vel)");
  PULSE_REQUIRE(s.heightfield != nullptr, "pulse_reset_terrain: plane terrain: a plane has no walkable table to spawn on");
  PULSE_REQUIRE(s.hf_rows >= 2 && s.hf_cols >= 2 && s.horizontal_scale > 0.0f, "pulse_reset_terrain: heightfield needs at least 2 x 2 cells "
                "and a positive horizontal_scale");
  PULSE_REQUIRE(s.center_points != nullptr && s.num_center_points >= 1 && s.num_center_points <= 32,
                "pulse_reset_terrain: num_center_points %lld outside [1, 32]", (long long)s.num_center_points);
  PULSE_REQUIRE(s.coord_x != nullptr && s.coord_y != nullptr && s.num_locations >= 1 && s.num_locations < (1ll << 32),
                "pulse_reset_terrain: walkable table of %lld locations (needs 1 .. 2^32 - 1)", (long long)s.num_locations);
  if (num_envs == 0) return PULSE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  reset_compact_kernel<<<1, kCompactThreads, 0, st>>>(a, (long long)num_envs);
  PULSE_LAUNCH_OK("reset_compact_kernel");
  const long long upper = (a.env_ids_in != nullptr ? a.num_ids : num_envs) * (a.amp_obs_buf != nullptr ? a.num_amp_steps : 1);
  terrain_reset_kernel<<<grid_for(upper, kResetWarps), kResetWarps * 32, 0, st>>>(lib->d, a, s);
  PULSE_LAUNCH_OK("terrain_reset_kernel");
  return PULSE_OK;
}
