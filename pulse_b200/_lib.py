"""ctypes binding of libpulse_b200.so -- the C ABI declared in include/pulse_b200.h.

There is no CPU fallback: if the library is missing the import fails loudly with build
instructions, and every compute call raises PulseError carrying pulse_last_error().
"""
import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libpulse_b200.so")


class PulseError(RuntimeError):
    pass


c_float_p = C.POINTER(C.c_float)
c_i64_p = C.POINTER(C.c_int64)
c_i32_p = C.POINTER(C.c_int32)
c_u8_p = C.POINTER(C.c_uint8)
c_f64_p = C.POINTER(C.c_double)


class MotionLibDesc(C.Structure):
    _fields_ = [
        ("gts", C.c_void_p), ("grs", C.c_void_p), ("lrs", C.c_void_p), ("gvs", C.c_void_p), ("gavs", C.c_void_p),
        ("dvs", C.c_void_p), ("motion_aa", C.c_void_p), ("lengths", C.c_void_p), ("dt", C.c_void_p),
        ("num_frames", C.c_void_p), ("length_starts", C.c_void_p), ("total_frames", C.c_int64),
        ("num_motions", C.c_int64), ("frame_rec", C.c_void_p), ("aux_rec", C.c_void_p),
    ]


class MotionQuery(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "motion_ids", "motion_times", "offset", "root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel",
        "motion_aa", "rg_pos", "rb_rot", "body_vel", "body_ang_vel", "frame_idx0", "frame_idx1", "blend")]


class ImStepArgs(C.Structure):
    _fields_ = [
        ("body_state", C.c_void_p), ("body_env_stride", C.c_int64),
        ("dof_vel", C.c_void_p), ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64),
        ("dof_force", C.c_void_p), ("dof_force_stride", C.c_int64), ("env_ids", C.c_void_p),
        ("progress_buf", C.c_void_p), ("motion_ids", C.c_void_p), ("motion_start_times", C.c_void_p),
        ("motion_start_offset", C.c_void_p), ("global_offset", C.c_void_p), ("cycle_counter", C.c_void_p),
        ("reset_buf_in", C.c_void_p), ("termination_distances", C.c_void_p),
        ("reset_body_mask", C.c_uint32), ("flags", C.c_uint32), ("dt", C.c_float),
        ("k_pos", C.c_float), ("k_rot", C.c_float), ("k_vel", C.c_float), ("k_ang_vel", C.c_float),
        ("w_pos", C.c_float), ("w_rot", C.c_float), ("w_vel", C.c_float), ("w_ang_vel", C.c_float),
        ("power_coefficient", C.c_float), ("cycle_motion", C.c_int32), ("max_episode_length", C.c_int64),
        ("enable_early_termination", C.c_int32), ("use_mean_reset", C.c_int32),
        ("obs_buf", C.c_void_p), ("obs_stride", C.c_int64), ("self_obs_buf", C.c_void_p), ("rew_buf", C.c_void_p),
        ("reward_raw", C.c_void_p), ("raw_stride", C.c_int64), ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p),
        ("pass_time", C.c_void_p), ("ref_body_pos", C.c_void_p), ("ref_body_vel", C.c_void_p),
        ("ref_body_rot", C.c_void_p), ("ref_dof_pos", C.c_void_p),
        ("env_count", C.c_void_p), ("recovery_counter", C.c_void_p), ("progress_rw", C.c_void_p), ("fdones_out", C.c_void_p),
    ]


class ImTrack(C.Structure):
    _fields_ = [("rank", C.c_int8 * 24), ("num_track", C.c_int32), ("version", C.c_int32)]


class ResetArgs(C.Structure):
    _fields_ = [
        ("reset_buf", C.c_void_p), ("env_ids_in", C.c_void_p), ("num_ids", C.c_int64), ("phase", C.c_void_p),
        ("seed", C.c_uint64), ("offset", C.c_uint64), ("motion_ids", C.c_void_p), ("motion_start_times", C.c_void_p),
        ("motion_start_offset", C.c_void_p), ("global_offset", C.c_void_p), ("cycle_counter", C.c_void_p), ("progress_buf", C.c_void_p),
        ("terminate_buf", C.c_void_p), ("root_states", C.c_void_p), ("root_env_stride", C.c_int64),
        ("dof_pos", C.c_void_p), ("dof_vel", C.c_void_p), ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64),
        ("rigid_body_state", C.c_void_p), ("body_env_stride", C.c_int64),
        ("contact_forces", C.c_void_p), ("contact_env_stride", C.c_int64), ("contact_bodies", C.c_int32),
        ("num_amp_steps", C.c_int32), ("amp_obs_buf", C.c_void_p), ("dt", C.c_float), ("reserved", C.c_int32),
        ("actor_ids", C.c_void_p), ("env_list", C.c_void_p), ("actor_list", C.c_void_p), ("count", C.c_void_p), ("amp_fresh", C.c_void_p),
        ("offset_dev", C.c_void_p),
    ]


class GetupResetArgs(C.Structure):
    _fields_ = [
        ("base", ResetArgs), ("recovery_u", C.c_void_p), ("fall_u", C.c_void_p), ("fall_keys", C.c_void_p),
        ("recovery_prob", C.c_float), ("fall_prob", C.c_float), ("recovery_steps", C.c_int32), ("reserved", C.c_int32),
        ("recovery_counter", C.c_void_p), ("available_fall_states", C.c_void_p), ("fall_id_assignments", C.c_void_p),
        ("fall_root_states", C.c_void_p), ("fall_root_stride", C.c_int64), ("fall_dof_pos", C.c_void_p), ("fall_dof_vel", C.c_void_p),
        ("fall_dof_env_stride", C.c_int64), ("fall_dof_elem_stride", C.c_int64), ("num_fall_states", C.c_int64),
        ("ref_list", C.c_void_p), ("fall_list", C.c_void_p), ("recovery_list", C.c_void_p), ("class_counts", C.c_void_p),
        ("env_class", C.c_void_p), ("error", C.c_void_p), ("fall_pick", C.c_void_p), ("fall_key_scratch", C.c_void_p),
    ]


class GetupAmpArgs(C.Structure):
    _fields_ = [
        ("body_state", C.c_void_p), ("body_env_stride", C.c_int64), ("dof_pos", C.c_void_p), ("dof_vel", C.c_void_p),
        ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64), ("amp_obs_buf", C.c_void_p), ("num_steps", C.c_int32),
        ("reserved", C.c_int32), ("fall_list", C.c_void_p), ("recovery_list", C.c_void_p), ("class_counts", C.c_void_p),
    ]


class WeightBlock(C.Structure):
    _fields_ = [("w", C.c_void_p), ("g", C.c_void_p), ("rows", C.c_int64), ("cols", C.c_int64), ("ld", C.c_int64), ("coef", C.c_float),
                ("reserved", C.c_int32), ("sumsq", C.c_void_p), ("sumsq2", C.c_void_p)]


class WeightReg(C.Structure):
    _fields_ = [("block", WeightBlock * 4), ("count", C.c_int32), ("reserved", C.c_int32)]


class PolicyPostArgs(C.Structure):
    _fields_ = [
        ("mu", C.c_void_p), ("ld_mu", C.c_int64), ("logstd", C.c_void_p), ("eps", C.c_void_p), ("ld_eps", C.c_int64),
        ("seed", C.c_uint64), ("rng_offset", C.c_void_p), ("rng_step", C.c_uint64), ("num_actions", C.c_int32), ("reserved", C.c_int32),
        ("actions", C.c_void_p), ("ld_actions", C.c_int64), ("neglogp", C.c_void_p), ("ld_neglogp", C.c_int64),
        ("mus_out", C.c_void_p), ("ld_mus", C.c_int64), ("value", C.c_void_p), ("ld_value", C.c_int64),
        ("value_mean", C.c_void_p), ("value_var", C.c_void_p), ("value_eps", C.c_float), ("reserved2", C.c_int32),
        ("values_out", C.c_void_p), ("ld_values", C.c_int64),
        ("pd_offset", C.c_void_p), ("pd_scale", C.c_void_p), ("pd_targets", C.c_void_p), ("ld_pd", C.c_int64),
    ]


class AmpRowArgs(C.Structure):
    _fields_ = [
        ("body_state", C.c_void_p), ("body_env_stride", C.c_int64), ("dof_pos", C.c_void_p), ("dof_vel", C.c_void_p),
        ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64), ("prev", C.c_void_p), ("ld_prev", C.c_int64),
        ("out", C.c_void_p), ("ld_out", C.c_int64), ("num_steps", C.c_int32), ("reserved", C.c_int32),
        ("fresh", C.c_void_p), ("fresh_rows", C.c_void_p), ("amp_width", C.c_int32), ("remove_base_rot", C.c_int32),
    ]


class AmpObsArgs(C.Structure):
    _fields_ = [
        ("body_state", C.c_void_p), ("body_env_stride", C.c_int64), ("dof_pos", C.c_void_p), ("dof_vel", C.c_void_p),
        ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64), ("amp_obs_buf", C.c_void_p),
        ("num_steps", C.c_int32), ("shift_history", C.c_int32),
    ]


class GaeArgs(C.Structure):
    _fields_ = [
        ("rewards", C.c_void_p), ("values", C.c_void_p), ("next_values", C.c_void_p), ("fdones", C.c_void_p),
        ("gamma", C.c_float), ("tau", C.c_float), ("advantages", C.c_void_p), ("returns", C.c_void_p), ("adv_sum", C.c_void_p),
    ]


class GemmEpilogue(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p), ("act", C.c_int32), ("gate_mode", C.c_int32), ("gate", C.c_void_p), ("ldg", C.c_int64),
        ("alpha", C.c_float), ("out", C.c_void_p), ("ldo", C.c_int64), ("out_t", C.c_void_p), ("ldot", C.c_int64),
        ("out_f32", C.c_void_p), ("ldf", C.c_int64), ("split_stride", C.c_int64), ("preact", C.c_void_p), ("ldp", C.c_int64),
        ("colsum", C.c_void_p), ("accumulate", C.c_int32), ("reserved", C.c_int32), ("sumsq", C.c_void_p),
        ("relu_mask", C.c_void_p), ("ld_rmask", C.c_int64), ("gate_mask", C.c_void_p), ("ld_gmask", C.c_int64),
    ]


GEMM_A_MN, GEMM_B_MN = 1, 2


class PpoLossArgs(C.Structure):
    _fields_ = [
        ("mu", C.c_void_p), ("ld_mu", C.c_int64), ("value", C.c_void_p), ("ld_value", C.c_int64), ("actions", C.c_void_p),
        ("old_neglogp", C.c_void_p), ("advantages", C.c_void_p), ("returns", C.c_void_p), ("old_mu", C.c_void_p),
        ("logstd", C.c_void_p), ("num_actions", C.c_int32), ("e_clip", C.c_float), ("critic_coef", C.c_float),
        ("bounds_coef", C.c_float), ("dmu", C.c_void_p), ("ld_dmu", C.c_int64), ("dmu_t", C.c_void_p), ("ld_dmu_t", C.c_int64),
        ("dvalue", C.c_void_p), ("ld_dv", C.c_int64), ("dvalue_t", C.c_void_p), ("ld_dv_t", C.c_int64), ("stats", C.c_void_p),
    ]


class VaeLatentArgs(C.Structure):
    _fields_ = [
        ("enc_head", C.c_void_p), ("ld_enc", C.c_int64), ("prior_head", C.c_void_p), ("ld_prior", C.c_int64),
        ("noise", C.c_void_p), ("ld_noise", C.c_int64), ("dz", C.c_void_p), ("ld_dz", C.c_int64), ("progress", C.c_void_p),
        ("latent", C.c_int32), ("horizon", C.c_int32), ("clamp", C.c_int32), ("reserved", C.c_int32),
        ("clamp_lo", C.c_float), ("clamp_hi", C.c_float), ("kld_coef", C.c_float), ("ar1_coef", C.c_float),
        ("regu_coef", C.c_float), ("phi", C.c_float),
        ("d_enc_head", C.c_void_p), ("ld_de", C.c_int64), ("d_prior_head", C.c_void_p), ("ld_dp", C.c_int64), ("stats", C.c_void_p),
    ]


class ReachStepArgs(C.Structure):
    _fields_ = [
        ("body_state", C.c_void_p), ("body_env_stride", C.c_int64), ("contact_forces", C.c_void_p), ("contact_env_stride", C.c_int64),
        ("termination_heights", C.c_void_p), ("tar_pos", C.c_void_p), ("progress_buf", C.c_void_p),
        ("contact_body_mask", C.c_uint32), ("reach_body_id", C.c_int32), ("enable_early_termination", C.c_int32), ("reserved", C.c_int32),
        ("max_episode_length", C.c_int64), ("obs_buf", C.c_void_p), ("obs_stride", C.c_int64), ("rew_buf", C.c_void_p),
        ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p),
    ]


class LoaderArgs(C.Structure):
    _fields_ = [
        ("pose_quat_global", C.c_void_p), ("root_trans", C.c_void_p), ("frame_clip", C.c_void_p), ("clip_start", C.c_void_p),
        ("fps", C.c_void_p), ("headings", C.c_void_p), ("parents", C.c_void_p), ("local_translation", C.c_void_p),
        ("total_frames", C.c_int64), ("num_clips", C.c_int64),
        ("gts", C.c_void_p), ("grs", C.c_void_p), ("lrs", C.c_void_p), ("gvs", C.c_void_p), ("gavs", C.c_void_p), ("dvs", C.c_void_p),
        ("tmp_vel", C.c_void_p), ("tmp_ang", C.c_void_p),
    ]


class ZTaskStepArgs(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("enable_early_termination", C.c_int32), ("body_state", C.c_void_p), ("body_env_stride", C.c_int64),
        ("contact_forces", C.c_void_p), ("contact_env_stride", C.c_int64), ("termination_heights", C.c_void_p),
        ("contact_body_mask", C.c_uint32), ("strike_body_mask", C.c_uint32), ("progress_buf", C.c_void_p), ("max_episode_length", C.c_int64),
        ("prev_root_pos", C.c_void_p), ("dt", C.c_float), ("power_coefficient", C.c_float), ("tar_speed", C.c_void_p),
        ("target_states", C.c_void_p), ("target_env_stride", C.c_int64), ("tar_contact_forces", C.c_void_p), ("tar_contact_env_stride", C.c_int64),
        ("dof_force", C.c_void_p), ("dof_force_stride", C.c_int64), ("dof_vel", C.c_void_p), ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64),
        ("obs_buf", C.c_void_p), ("obs_stride", C.c_int64), ("rew_buf", C.c_void_p), ("reward_raw", C.c_void_p), ("raw_stride", C.c_int64),
        ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p),
    ]


ZTASK_SPEED, ZTASK_STRIKE, ZTASK_REACH = 1, 2, 3
ZPOSE_AS_IS, ZPOSE_ROOT_XY_ZERO, ZPOSE_FACE_X = 0, 1, 2
ZINIT_RANDOM, ZINIT_START = 0, 1


class ZTaskResetArgs(C.Structure):
    _fields_ = [
        ("reset_buf", C.c_void_p), ("env_ids_in", C.c_void_p), ("num_ids", C.c_int64), ("motion_ids_in", C.c_void_p), ("motion_u", C.c_void_p), ("phase", C.c_void_p),
        ("strike_u", C.c_void_p), ("sampling_cdf", C.c_void_p), ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", C.c_void_p),
        ("floor", C.c_void_p), ("floor_len", C.c_int64), ("pose_mode", C.c_int32), ("upright", C.c_int32), ("state_init", C.c_int32),
        ("amp_width", C.c_int32), ("num_amp_steps", C.c_int32), ("dt", C.c_float), ("amp_obs_buf", C.c_void_p),
        ("sampled_motion_ids", C.c_void_p), ("motion_start_times", C.c_void_p), ("progress_buf", C.c_void_p), ("terminate_buf", C.c_void_p),
        ("root_states", C.c_void_p), ("root_env_stride", C.c_int64), ("dof_pos", C.c_void_p), ("dof_vel", C.c_void_p),
        ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64), ("rigid_body_state", C.c_void_p), ("body_env_stride", C.c_int64),
        ("contact_forces", C.c_void_p), ("contact_env_stride", C.c_int64), ("contact_bodies", C.c_int32), ("reserved", C.c_int32),
        ("target_states", C.c_void_p), ("target_env_stride", C.c_int64), ("near_prob", C.c_float), ("near_dist", C.c_float),
        ("tar_dist_min", C.c_float), ("tar_dist_max", C.c_float), ("actor_ids", C.c_void_p), ("tar_actor_ids", C.c_void_p),
        ("env_list", C.c_void_p), ("actor_list", C.c_void_p), ("tar_actor_list", C.c_void_p), ("count", C.c_void_p), ("amp_fresh", C.c_void_p),
    ]


PLANE_DEMO_CLIP, PLANE_DEMO_TIME, PLANE_REPLAY_KEEP, PLANE_REPLAY_SUBSET, PLANE_RING_PERM = 5, 6, 7, 8, 9
RING_HEAD, RING_TOTAL, RING_SAMPLE_HEAD, RING_PERM_KEY, RING_DRAWS, RING_LAST_COUNT, RING_CTRS = 0, 1, 2, 3, 4, 5, 8


class AmpRing(C.Structure):
    _fields_ = [("rows", C.c_void_p), ("capacity", C.c_int64), ("ctr", C.c_void_p), ("seed", C.c_uint64), ("row_floats", C.c_int32),
                ("reserved", C.c_int32)]


class AmpDemoArgs(C.Structure):
    _fields_ = [("ring", AmpRing), ("sampling_cdf", C.c_void_p), ("num_samples", C.c_int64), ("num_steps", C.c_int32), ("amp_width", C.c_int32),
                ("upright", C.c_int32), ("dt", C.c_float), ("motion_ids_out", C.c_void_p), ("times_out", C.c_void_p)]


class AmpStoreArgs(C.Structure):
    _fields_ = [("ring", AmpRing), ("src", C.c_void_p), ("num_rows", C.c_int64), ("keep_prob", C.c_float), ("reserved", C.c_int32),
                ("kept", C.c_void_p), ("src_rows_out", C.c_void_p)]


class AmpSampleArgs(C.Structure):
    _fields_ = [("ring", AmpRing), ("n", C.c_int64), ("block", C.c_int64), ("take", C.c_int64), ("fallback", C.c_void_p), ("out", C.c_void_p),
                ("ring_rows_out", C.c_void_p)]


class ZTaskTaskArgs(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("reserved", C.c_int32), ("env_list", C.c_void_p), ("count", C.c_void_p), ("rand", C.c_void_p),
        ("steps_in", C.c_void_p), ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", C.c_void_p), ("progress_buf", C.c_void_p),
        ("change_steps", C.c_void_p), ("tar_pos", C.c_void_p), ("tar_speed", C.c_void_p), ("dist_max", C.c_float), ("height_scale", C.c_float),
        ("height_min", C.c_float), ("speed_scale", C.c_float), ("speed_min", C.c_float), ("reserved2", C.c_int32),
        ("steps_min", C.c_int64), ("steps_max", C.c_int64),
    ]


class LatentPostArgs(C.Structure):
    _fields_ = [
        ("mu", C.c_void_p), ("ld_mu", C.c_int64), ("logstd", C.c_void_p), ("eps", C.c_void_p), ("ld_eps", C.c_int64),
        ("seed", C.c_uint64), ("rng_offset", C.c_void_p), ("rng_step", C.c_uint64), ("latent", C.c_int32), ("reserved", C.c_int32),
        ("actions", C.c_void_p), ("ld_actions", C.c_int64), ("neglogp", C.c_void_p), ("ld_neglogp", C.c_int64),
        ("value", C.c_void_p), ("ld_value", C.c_int64), ("value_mean", C.c_void_p), ("value_var", C.c_void_p), ("value_eps", C.c_float),
        ("reserved2", C.c_int32), ("values_out", C.c_void_p), ("ld_values", C.c_int64), ("prior_mu", C.c_void_p), ("ld_prior", C.c_int64),
        ("z_bf16", C.c_void_p), ("ld_z", C.c_int64),
    ]


class ZTaskPrePhysicsArgs(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("dofs", C.c_int32), ("action", C.c_void_p), ("ld_action", C.c_int64), ("pd_offset", C.c_void_p),
        ("pd_scale", C.c_void_p), ("freeze", C.c_void_p), ("pd_out", C.c_void_p), ("ld_pd", C.c_int64), ("root_states", C.c_void_p),
        ("root_env_stride", C.c_int64), ("prev_root_pos", C.c_void_p), ("progress_buf", C.c_void_p), ("change_steps", C.c_void_p),
        ("tar_pos", C.c_void_p), ("tar_speed", C.c_void_p), ("rand", C.c_void_p), ("steps_in", C.c_void_p), ("seed", C.c_uint64),
        ("offset", C.c_uint64), ("offset_dev", C.c_void_p), ("dist_max", C.c_float), ("height_min", C.c_float), ("height_max", C.c_float),
        ("speed_scale", C.c_float), ("speed_min", C.c_float), ("reserved", C.c_int32), ("steps_min", C.c_int64), ("steps_max", C.c_int64),
    ]


class SmplxMotionLibDesc(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "lengths", "dt", "num_frames", "length_starts")] + [
        ("total_frames", C.c_int64), ("num_motions", C.c_int64), ("frame_rec", C.c_void_p), ("aux_rec", C.c_void_p)]


class SmplxMotionQuery(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "motion_ids", "motion_times", "offset", "root_pos", "root_rot", "root_vel", "root_ang_vel", "dof_pos", "dof_vel", "rg_pos", "rb_rot",
        "body_vel", "body_ang_vel")]


class SmplxSpeedStepArgs(C.Structure):
    _fields_ = [
        ("enable_early_termination", C.c_int32), ("reserved", C.c_int32), ("body_state", C.c_void_p), ("body_env_stride", C.c_int64),
        ("contact_forces", C.c_void_p), ("contact_env_stride", C.c_int64), ("termination_heights", C.c_void_p), ("contact_body_mask", C.c_uint64),
        ("progress_buf", C.c_void_p), ("max_episode_length", C.c_int64), ("prev_root_pos", C.c_void_p), ("dt", C.c_float), ("reserved2", C.c_float),
        ("tar_speed", C.c_void_p), ("obs_buf", C.c_void_p), ("obs_stride", C.c_int64), ("rew_buf", C.c_void_p), ("reward_raw", C.c_void_p),
        ("raw_stride", C.c_int64), ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p),
    ]


class SmplxTargetStepArgs(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("enable_early_termination", C.c_int32), ("body_state", C.c_void_p), ("body_env_stride", C.c_int64),
        ("contact_forces", C.c_void_p), ("contact_env_stride", C.c_int64), ("termination_heights", C.c_void_p), ("contact_body_mask", C.c_uint64),
        ("strike_body_mask", C.c_uint64), ("reach_body_id", C.c_int32), ("reserved", C.c_int32), ("progress_buf", C.c_void_p),
        ("max_episode_length", C.c_int64), ("tar_pos", C.c_void_p), ("prev_root_pos", C.c_void_p), ("dt", C.c_float), ("reserved2", C.c_float),
        ("target_states", C.c_void_p), ("target_env_stride", C.c_int64), ("tar_contact_forces", C.c_void_p), ("tar_contact_env_stride", C.c_int64),
        ("obs_buf", C.c_void_p), ("obs_stride", C.c_int64), ("rew_buf", C.c_void_p), ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p),
    ]


SMPLX_BODIES, SMPLX_DOF, SMPLX_SELF_OBS, SMPLX_SPEED_OBS = 52, 153, 778, 781
SMPLX_REACH_OBS, SMPLX_STRIKE_OBS = 781, 793          # PULSE_SMPLX_REACH_OBS / PULSE_SMPLX_STRIKE_OBS: 778 + 3 / + 15
SMPLX_AMP_OBS, SMPLX_AMP_OBS_NO_HEIGHT = 466, 465       # PULSE_SMPLX_AMP_OBS(_NO_HEIGHT): the SMPL-X AMP row, with / without root height


# Philox index planes of the latent tasks' draws (include/pulse_b200.h): index = env + plane
ZTASK_PLANE_RESET, ZTASK_PLANE_STRIKE, ZTASK_PLANE_RESET_TASK, ZTASK_PLANE_UPDATE_TASK = 0, 1 << 32, 2 << 32, 3 << 32


class TerrainStepArgs(C.Structure):
    _fields_ = [
        ("flags", C.c_uint32), ("upright", C.c_int32), ("body_state", C.c_void_p), ("body_env_stride", C.c_int64),
        ("root_states", C.c_void_p), ("root_env_stride", C.c_int64), ("progress_buf", C.c_void_p), ("max_episode_length", C.c_int64),
        ("contact_forces", C.c_void_p), ("contact_env_stride", C.c_int64), ("contact_body_mask", C.c_uint32),
        ("enable_early_termination", C.c_int32), ("no_collision_check", C.c_int32), ("fuzzy_target", C.c_int32), ("power_reward", C.c_int32),
        ("num_traj_samples", C.c_int32), ("num_height_points", C.c_int32), ("num_center_points", C.c_int32), ("head_body_id", C.c_int32),
        ("use_center_height", C.c_int32), ("dt", C.c_float), ("traj_dur", C.c_float), ("traj_sample_timestep", C.c_float),
        ("fail_dist", C.c_float), ("power_coefficient", C.c_float), ("traj_verts", C.c_void_p),
        ("heightfield", C.c_void_p), ("hf_rows", C.c_int64), ("hf_cols", C.c_int64), ("horizontal_scale", C.c_float), ("vertical_scale", C.c_float),
        ("height_points", C.c_void_p), ("center_points", C.c_void_p), ("dof_force", C.c_void_p), ("dof_force_stride", C.c_int64),
        ("dof_vel", C.c_void_p), ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64), ("env_ids", C.c_void_p), ("env_count", C.c_void_p),
        ("obs_buf", C.c_void_p), ("obs_stride", C.c_int64), ("rew_buf", C.c_void_p), ("reward_raw", C.c_void_p), ("raw_stride", C.c_int64),
        ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p),
    ]


class TrajResetArgs(C.Structure):
    _fields_ = [
        ("env_ids", C.c_void_p), ("num_ids", C.c_int64), ("init_pos", C.c_void_p), ("init_stride", C.c_int64), ("rand", C.c_void_p),
        ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", C.c_void_p), ("dtheta_scale", C.c_float), ("dspeed_scale", C.c_float),
        ("seg_dt", C.c_float), ("speed_min", C.c_float), ("speed_max", C.c_float), ("sharp_turn_prob", C.c_float), ("verts", C.c_void_p),
    ]


class TerrainHeightsArgs(C.Structure):
    _fields_ = [
        ("mode", C.c_int32), ("upright", C.c_int32), ("root_states", C.c_void_p), ("root_stride", C.c_int64), ("num_rows", C.c_int64),
        ("points", C.c_void_p), ("num_points", C.c_int64), ("heightfield", C.c_void_p), ("hf_rows", C.c_int64), ("hf_cols", C.c_int64),
        ("horizontal_scale", C.c_float), ("vertical_scale", C.c_float), ("heights", C.c_void_p), ("heights_stride", C.c_int64),
    ]


TRAJ_VERTS = 101
TRAJ_DRAWS = 4 * (TRAJ_VERTS - 1) + 2
HEIGHTS_CENTER, HEIGHTS_GRID = 1, 2


class TrajListArgs(C.Structure):
    _fields_ = [
        ("env_list", C.c_void_p), ("count", C.c_void_p), ("root_states", C.c_void_p), ("root_env_stride", C.c_int64), ("rand", C.c_void_p),
        ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", C.c_void_p), ("dtheta_scale", C.c_float), ("dspeed_scale", C.c_float),
        ("seg_dt", C.c_float), ("speed_min", C.c_float), ("speed_max", C.c_float), ("sharp_turn_prob", C.c_float), ("verts", C.c_void_p),
    ]


class TerrainSpawnArgs(C.Structure):
    _fields_ = [
        ("heightfield", C.c_void_p), ("hf_rows", C.c_int64), ("hf_cols", C.c_int64), ("horizontal_scale", C.c_float), ("vertical_scale", C.c_float),
        ("center_points", C.c_void_p), ("num_center_points", C.c_int64), ("coord_x", C.c_void_p), ("coord_y", C.c_void_p),
        ("num_locations", C.c_int64), ("loc_ids_in", C.c_void_p), ("loc_ids_out", C.c_void_p),
    ]


TRAJ_LIST_PLANE = 4 << 32      # Philox index plane of pulse_traj_reset_list: index = env + TRAJ_LIST_PLANE


def traj_list_philox_blocks(env: int, offset: int, offset_dev: int = 0):
    """The Philox4x32-10 blocks (index, counters) one `pulse_traj_reset_list` reset of `env` reads, as the kernel keys them:
    index env + 4 * 2^32, counters TRAJ_VERTS * (offset + offset_dev) + k for k in [0, TRAJ_VERTS)."""
    base = (TRAJ_VERTS * ((offset + offset_dev) % 2 ** 64)) % 2 ** 64
    return env + TRAJ_LIST_PLANE, [(base + k) % 2 ** 64 for k in range(TRAJ_VERTS)]


class TaskObsArgs(C.Structure):
    _fields_ = [
        ("body_state", C.c_void_p), ("body_env_stride", C.c_int64), ("track_ids", C.c_void_p),
        ("num_track", C.c_int32), ("time_steps", C.c_int32), ("version", C.c_int32), ("upright", C.c_int32),
        ("ref_pos", C.c_void_p), ("ref_rot", C.c_void_p), ("ref_vel", C.c_void_p), ("ref_ang_vel", C.c_void_p),
        ("dof_pos", C.c_void_p), ("dof_env_stride", C.c_int64), ("dof_elem_stride", C.c_int64), ("ref_dof_pos", C.c_void_p),
        ("obs", C.c_void_p), ("obs_stride", C.c_int64), ("num_envs", C.c_int64),
    ]


class EvalArgs(C.Structure):
    _fields_ = [
        ("body_pos", C.c_void_p), ("pos_env_stride", C.c_int64), ("pos_body_stride", C.c_int64),
        ("body_pos_gt", C.c_void_p), ("gt_env_stride", C.c_int64), ("gt_body_stride", C.c_int64),
        ("terminate", C.c_void_p), ("num_steps", C.c_void_p),
        ("num_envs", C.c_int32), ("bound", C.c_int32), ("max_steps_all", C.c_int32), ("reserved", C.c_int32),
        ("ctrl", C.c_void_p), ("terminate_state", C.c_void_p), ("hist", C.c_void_p), ("sums", C.c_void_p), ("counts", C.c_void_p),
        ("mpjpe_out", C.c_void_p),
    ]


PEER_MAX, PEER_MAX_GRID, PEER_SIGNAL_BYTES = 8, 256, 3 * 8 * 4 + 8 * 8


class PeerAdamArgs(C.Structure):
    _fields_ = [
        ("rank", C.c_int32), ("world", C.c_int32),
        ("grads", C.c_void_p * PEER_MAX), ("params", C.c_void_p * PEER_MAX), ("params_bf16", C.c_void_p * PEER_MAX),
        ("signals", C.c_void_p * PEER_MAX),
        ("mc_grads", C.c_void_p), ("mc_params", C.c_void_p), ("mc_params_bf16", C.c_void_p),
        ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("count", C.c_int64),
        ("max_norm", C.c_float), ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("grid", C.c_int32),
        ("timeout_ms", C.c_uint32), ("reserved", C.c_uint32), ("step", C.c_void_p), ("epoch", C.c_void_p), ("cta_partials", C.c_void_p), ("grid_bar", C.c_void_p),
    ]


ABI_VERSION = 3
HEAD1_MAX_CTAS = 264        # PULSE_HEAD1_MAX_CTAS: rows of the pulse_head1_backward partial-sum scratch
ACT_NONE, ACT_RELU, ACT_SILU = 0, 1, 2
Z_SAMPLE, Z_MEAN, Z_RESIDUAL = 0, 1, 2
STEP_REWARD, STEP_RESET, STEP_OBS, STEP_ALL, STEP_ADVANCE = 1, 2, 4, 7, 8
GETUP_REF, GETUP_FALL, GETUP_RECOVERY = 1, 2, 3

# name -> (restype, argtypes); mirrors include/pulse_b200.h one to one
SIGNATURES = {
    "pulse_abi_version": (C.c_int, []),
    "pulse_last_error": (C.c_char_p, []),
    "pulse_launch_count": (C.c_int64, []),
    "pulse_motionlib_create": (C.c_int, [C.POINTER(MotionLibDesc), C.c_void_p, C.POINTER(C.c_void_p)]),
    "pulse_motionlib_destroy": (C.c_int, [C.c_void_p]),
    "pulse_motion_state": (C.c_int, [C.c_void_p, C.POINTER(MotionQuery), C.c_int64, C.c_void_p]),
    "pulse_im_step": (C.c_int, [C.c_void_p, C.POINTER(ImStepArgs), C.c_int64, C.c_void_p]),
    "pulse_im_track_step": (C.c_int, [C.c_void_p, C.POINTER(ImStepArgs), C.POINTER(ImTrack), C.c_int64, C.c_void_p]),
    "pulse_reset_ref_state": (C.c_int, [C.c_void_p, C.POINTER(ResetArgs), C.c_int64, C.c_void_p]),
    "pulse_reset_getup": (C.c_int, [C.c_void_p, C.POINTER(GetupResetArgs), C.c_int64, C.c_void_p]),
    "pulse_getup_amp_init": (C.c_int, [C.POINTER(GetupAmpArgs), C.c_int64, C.c_void_p]),
    "pulse_policy_post": (C.c_int, [C.POINTER(PolicyPostArgs), C.c_int64, C.c_void_p]),
    "pulse_value_post": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "pulse_amp_obs_row": (C.c_int, [C.POINTER(AmpRowArgs), C.c_int64, C.c_void_p]),
    "pulse_bump_counter": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p]),
    "pulse_event_create": (C.c_int, [C.POINTER(C.c_void_p)]),
    "pulse_event_destroy": (C.c_int, [C.c_void_p]),
    "pulse_event_record": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pulse_event_elapsed_ms": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]),
    "pulse_amp_obs": (C.c_int, [C.POINTER(AmpObsArgs), C.c_int64, C.c_void_p]),
    "pulse_gae": (C.c_int, [C.POINTER(GaeArgs), C.c_int32, C.c_int64, C.c_void_p]),
    "pulse_normalize_advantages": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_gemm_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                  C.POINTER(GemmEpilogue), C.c_int32, C.c_uint32, C.c_void_p]),
    "pulse_gemm_num_splits": (C.c_int, [C.c_int64, C.c_int32]),
    "pulse_gemm_tile_n": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32]),
    "pulse_gemm_last_launch": (C.c_int, [C.POINTER(C.c_int32)]),
    "pulse_gemm_last_tile_n": (C.c_int, []),
    "pulse_normalize_to_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_int64, C.c_float, C.c_void_p]),
    "pulse_normalize_moments": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_float, C.c_void_p]),
    "pulse_normalize_split": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pulse_head1_forward": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_head1_backward": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pulse_ordered_sum_add": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_column_moments": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "pulse_rms_merge": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p,
                                  C.c_void_p]),
    "pulse_gaussian_sample": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "pulse_ppo_loss": (C.c_int, [C.POINTER(PpoLossArgs), C.c_int64, C.c_void_p]),
    "pulse_disc_loss": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_float, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pulse_relu_mask_scale": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_weight_reg": (C.c_int, [C.POINTER(WeightReg), C.c_void_p]),
    "pulse_axpy": (C.c_int, [C.c_float, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_column_sum_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "pulse_reduce_slabs": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "pulse_sum_squares": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pulse_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_float,
                                  C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "pulse_peer_reduce_adam": (C.c_int, [C.POINTER(PeerAdamArgs), C.c_void_p]),
    "pulse_refresh_weight_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_normalize_cols": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int64,
                                       C.c_int64, C.c_void_p]),
    "pulse_copy_cols_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_vae_reparam": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                    C.c_float, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_vae_reparam_philox": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_uint64,
                                           C.c_void_p, C.c_uint64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_distill_pre_physics": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                            C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pulse_vae_action_loss": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_int64,
                                        C.c_void_p, C.c_void_p]),
    "pulse_vae_latent_loss": (C.c_int, [C.POINTER(VaeLatentArgs), C.c_int64, C.c_void_p]),
    "pulse_pnn_compose": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                    C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_pd_targets": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64,
                                   C.c_void_p]),
    "pulse_reach_update_task": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float,
                                          C.c_int64, C.c_void_p]),
    "pulse_reach_step": (C.c_int, [C.POINTER(ReachStepArgs), C.c_int64, C.c_void_p]),
    "pulse_ztask_step": (C.c_int, [C.POINTER(ZTaskStepArgs), C.c_int64, C.c_void_p]),
    "pulse_reach_obs_list": (C.c_int, [C.POINTER(ReachStepArgs), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_ztask_obs_list": (C.c_int, [C.POINTER(ZTaskStepArgs), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_reset_ztask": (C.c_int, [C.c_void_p, C.POINTER(ZTaskResetArgs), C.c_int64, C.c_void_p]),
    "pulse_ztask_reset_task": (C.c_int, [C.POINTER(ZTaskTaskArgs), C.c_int64, C.c_void_p]),
    "pulse_latent_post": (C.c_int, [C.POINTER(LatentPostArgs), C.c_int64, C.c_void_p]),
    "pulse_ztask_pre_physics": (C.c_int, [C.POINTER(ZTaskPrePhysicsArgs), C.c_int64, C.c_void_p]),
    "pulse_reach_rollout_step": (C.c_int, [C.POINTER(ReachStepArgs), C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_ztask_rollout_step": (C.c_int, [C.POINTER(ZTaskStepArgs), C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_terrain_step": (C.c_int, [C.POINTER(TerrainStepArgs), C.c_int64, C.c_void_p]),
    "pulse_terrain_rollout_step": (C.c_int, [C.POINTER(TerrainStepArgs), C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_traj_reset": (C.c_int, [C.POINTER(TrajResetArgs), C.c_void_p]),
    "pulse_terrain_heights": (C.c_int, [C.POINTER(TerrainHeightsArgs), C.c_void_p]),
    "pulse_traj_reset_list": (C.c_int, [C.POINTER(TrajListArgs), C.c_int64, C.c_void_p]),
    "pulse_reset_terrain": (C.c_int, [C.c_void_p, C.POINTER(ZTaskResetArgs), C.POINTER(TerrainSpawnArgs), C.c_int64, C.c_void_p]),
    "pulse_task_obs_size": (C.c_int, [C.c_int32, C.c_int32, C.c_int32]),
    "pulse_im_task_obs": (C.c_int, [C.POINTER(TaskObsArgs), C.c_void_p]),
    "pulse_eval_step": (C.c_int, [C.POINTER(EvalArgs), C.c_void_p]),
    "pulse_motionlib_load_clips": (C.c_int, [C.POINTER(LoaderArgs), C.c_void_p]),
    "pulse_smplx_motionlib_create": (C.c_int, [C.POINTER(SmplxMotionLibDesc), C.c_void_p, C.POINTER(C.c_void_p)]),
    "pulse_smplx_motionlib_destroy": (C.c_int, [C.c_void_p]),
    "pulse_smplx_motion_state": (C.c_int, [C.c_void_p, C.POINTER(SmplxMotionQuery), C.c_int64, C.c_void_p]),
    "pulse_smplx_speed_step": (C.c_int, [C.POINTER(SmplxSpeedStepArgs), C.c_int64, C.c_void_p]),
    "pulse_smplx_speed_obs_list": (C.c_int, [C.POINTER(SmplxSpeedStepArgs), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_smplx_speed_rollout_step": (C.c_int, [C.POINTER(SmplxSpeedStepArgs), C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_reset_ztask_smplx": (C.c_int, [C.c_void_p, C.POINTER(ZTaskResetArgs), C.c_int64, C.c_void_p]),
    "pulse_smplx_target_step": (C.c_int, [C.POINTER(SmplxTargetStepArgs), C.c_int64, C.c_void_p]),
    "pulse_smplx_target_obs_list": (C.c_int, [C.POINTER(SmplxTargetStepArgs), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_smplx_target_rollout_step": (C.c_int, [C.POINTER(SmplxTargetStepArgs), C.c_void_p, C.c_int64, C.c_void_p]),
    "pulse_reset_smplx_target": (C.c_int, [C.c_void_p, C.POINTER(ZTaskResetArgs), C.c_int64, C.c_void_p]),
    "pulse_smplx_amp_obs_row": (C.c_int, [C.POINTER(AmpRowArgs), C.c_int64, C.c_void_p]),
    "pulse_amp_demo_fetch": (C.c_int, [C.c_void_p, C.POINTER(AmpDemoArgs), C.c_void_p]),
    "pulse_smplx_amp_demo_fetch": (C.c_int, [C.c_void_p, C.POINTER(AmpDemoArgs), C.c_void_p]),
    "pulse_amp_replay_store": (C.c_int, [C.POINTER(AmpStoreArgs), C.c_void_p]),
    "pulse_amp_ring_sample": (C.c_int, [C.POINTER(AmpSampleArgs), C.c_void_p]),
}

_lib = None


def load():
    """Loads the shared library (once). Raises PulseError with build instructions if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PulseError(f"{LIB_PATH} is missing: build it with `python -m pulse_b200.build` "
                         "(nvcc, sm_90a). pulse_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.pulse_abi_version() != ABI_VERSION:
        raise PulseError(f"ABI version mismatch: library {lib.pulse_abi_version()} != binding {ABI_VERSION}")
    _lib = lib
    return lib


def check(status, what):
    if status != 0:
        msg = load().pulse_last_error().decode("utf-8", "replace")
        raise PulseError(f"{what} failed with status {status}: {msg}")


GEMM_LAUNCH_FIELDS = ("mode", "stages", "tile_n", "tma_out", "splits", "grid")


def gemm_last_launch() -> dict:
    """The kernel the last GEMM launch from the host took (pulse_gemm_last_launch), by field name; all 0 before the first."""
    out = (C.c_int32 * len(GEMM_LAUNCH_FIELDS))()
    check(load().pulse_gemm_last_launch(out), "pulse_gemm_last_launch")
    return dict(zip(GEMM_LAUNCH_FIELDS, out))


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def current_stream(device=None):
    import torch
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class GraphEvent:
    """CUDA event recorded with cudaEventRecordExternal: usable for timing INSIDE captured CUDA graphs (every replay re-records it)."""

    def __init__(self):
        self._h = C.c_void_p()
        check(load().pulse_event_create(C.byref(self._h)), "pulse_event_create")

    def record(self, device=None):
        check(load().pulse_event_record(self._h, current_stream(device)), "pulse_event_record")

    def elapsed_ms(self, stop: "GraphEvent") -> float:
        ms = C.c_float()
        check(load().pulse_event_elapsed_ms(self._h, stop._h, C.byref(ms)), "pulse_event_elapsed_ms")
        return float(ms.value)

    def __del__(self):
        try:
            if self._h:
                load().pulse_event_destroy(self._h)
        except Exception:
            pass
