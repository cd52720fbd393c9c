"""CPU oracle for the PULSE hot path (TEST INFRASTRUCTURE -- never imported by pulse_b200/).

A standalone fp32 PyTorch-CPU restatement of the arithmetic of the reference's per-step rollout and
update path, written from the behaviour of the reference functions cited beside each routine
(paths relative to the reference tree).  It exists so that the CUDA path can be checked on a GPU box
where the reference itself is not present, and so `bench.py` has a CPU arm (`cpu_baseline`,
`--impl reference`, kind "port") that does the same work the reference's PyTorch path does.

Pinning: `tests/test_oracle_vs_golden.py` checks every routine here against `tests/golden/*.npz`,
which `tests/golden/make_golden.py` produced by running the reference's own functions (imported
unmodified from the reference tree under `oracle/refshim`); `make_golden_reference_pins.py` adds the
reference's outputs on fresh seeded inputs.  Integer outputs (frame indices, reset / terminate
masks) must be identical; float outputs agree to 1e-6 or better (same op order, same library).

Third-party arithmetic absent from the reference tree and restated here [3P-memory]:
  * isaacgym.torch_utils (Isaac Gym Preview 4, unpinned): quat_mul (8-product form), quat_conjugate,
    quat_from_angle_axis, normalize, normalize_angle.
  * rl_games 1.1.4 (requirement.txt:27): ModelA2CContinuousLogStd neglogp / entropy,
    torch_ext.policy_kl, swap_and_flatten01.

Only tests/, __graft_entry__.smoke() and bench.py's CPU arms may import this module.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional, Tuple

import torch

F32 = torch.float32
NUM_BODIES = 24
NUM_DOF = 69
SELF_OBS = 358
TASK_OBS_V6 = 576
AMP_OBS = 196
# dof columns dropped by the AMP "dof_subset" (L_Toe, R_Toe, L_Hand, R_Hand) -- humanoid.py:397,417-421
AMP_DROPPED_JOINTS = (3, 7, 17, 22)  # joint index = body index - 1
KEY_BODY_IDS = (7, 3, 22, 17)  # R_Ankle, L_Ankle, R_Wrist, L_Wrist -- env_im.yaml:36
RESET_BODY_IDS = tuple(j for j in range(24) if j not in (3, 4, 7, 8))  # env_im.yaml:38
# dt = control_freq_inv * sim dt = 2 * fp32(1/60) -> fp32(1/30)  (humanoid.py:122, config.py:47)
STEP_DT = float(torch.tensor(1.0 / 60.0, dtype=F32) * 2)


# ------------------------------------------------------------------------------------------------
# quaternion primitives (xyzw)
# ------------------------------------------------------------------------------------------------
def quat_mul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """isaacgym.torch_utils.quat_mul [3P-memory]: Hamilton product, 8-multiplication form."""
    x1, y1, z1, w1 = a.unbind(-1)
    x2, y2, z2, w2 = b.unbind(-1)
    ww = (z1 + x1) * (x2 + y2)
    yy = (w1 - y1) * (w2 + z2)
    zz = (w1 + y1) * (w2 - z2)
    xx = ww + yy + zz
    qq = 0.5 * (xx + (z1 - x1) * (x2 - y2))
    w = qq - ww + (z1 - y1) * (y2 - z2)
    x = qq - xx + (x1 + w1) * (x2 + w2)
    y = qq - yy + (w1 - x1) * (y2 + z2)
    z = qq - zz + (z1 + y1) * (w2 - x2)
    return torch.stack([x, y, z, w], dim=-1)


def quat_conj(q: torch.Tensor) -> torch.Tensor:
    """isaacgym.torch_utils.quat_conjugate [3P-memory]."""
    return torch.cat([-q[..., :3], q[..., 3:]], dim=-1)


def _unit(x: torch.Tensor, eps: float = 1e-9) -> torch.Tensor:
    """isaacgym.torch_utils.normalize [3P-memory]: x / max(|x|, eps)."""
    return x / x.norm(p=2, dim=-1).clamp(min=eps).unsqueeze(-1)


def quat_rotate(q: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """phc/utils/torch_utils.py:45-55 (my_quat_rotate), any leading shape."""
    w = q[..., 3:4]
    u = q[..., :3]
    a = v * (2.0 * w ** 2 - 1.0)
    b = torch.cross(u, v, dim=-1) * w * 2.0
    c = u * (u * v).sum(-1, keepdim=True) * 2.0
    return a + b + c


def wrap_angle(x: torch.Tensor) -> torch.Tensor:
    """isaacgym.torch_utils.normalize_angle [3P-memory]."""
    return torch.atan2(torch.sin(x), torch.cos(x))


def quat_from_angle_axis(angle: torch.Tensor, axis: torch.Tensor) -> torch.Tensor:
    """isaacgym.torch_utils.quat_from_angle_axis [3P-memory]."""
    half = (angle / 2).unsqueeze(-1)
    return _unit(torch.cat([_unit(axis) * half.sin(), half.cos()], dim=-1))


def quat_to_angle_axis(q: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """phc/utils/torch_utils.py:57-78."""
    w = q[..., 3]
    s = torch.sqrt(1 - w * w)
    ang = wrap_angle(2 * torch.acos(w))
    axis = q[..., :3] / s.unsqueeze(-1)
    ok = s.abs() > 1e-5
    z_axis = torch.zeros_like(axis)
    z_axis[..., 2] = 1
    ang = torch.where(ok, ang, torch.zeros_like(ang))
    axis = torch.where(ok.unsqueeze(-1), axis, z_axis)
    return ang, axis


def quat_to_exp_map(q: torch.Tensor) -> torch.Tensor:
    """phc/utils/torch_utils.py:81-97."""
    ang, axis = quat_to_angle_axis(q)
    return ang.unsqueeze(-1) * axis


def exp_map_to_quat(e: torch.Tensor) -> torch.Tensor:
    """phc/utils/torch_utils.py:148-172."""
    ang = e.norm(dim=-1)
    axis = e / ang.unsqueeze(-1)
    ang = wrap_angle(ang)
    ok = ang.abs() > 1e-5
    z_axis = torch.zeros_like(e)
    z_axis[..., 2] = 1
    ang = torch.where(ok, ang, torch.zeros_like(ang))
    axis = torch.where(ok.unsqueeze(-1), axis, z_axis)
    return quat_from_angle_axis(ang, axis)


def quat_to_six(q: torch.Tensor) -> torch.Tensor:
    """phc/utils/torch_utils.py:100-113 (quat_to_tan_norm): rotated x-axis then rotated z-axis."""
    ex = torch.zeros_like(q[..., :3])
    ex[..., 0] = 1
    ez = torch.zeros_like(q[..., :3])
    ez[..., 2] = 1
    return torch.cat([quat_rotate(q, ex), quat_rotate(q, ez)], dim=-1)


def slerp(q0: torch.Tensor, q1: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    """phc/utils/torch_utils.py:175-197.  `t` broadcasts against [...,1]; result not renormalised."""
    c = (q0 * q1).sum(-1)
    q1 = torch.where((c < 0).unsqueeze(-1), -q1, q1)
    c = c.abs().unsqueeze(-1)
    half = torch.acos(c)
    s = torch.sqrt(1.0 - c * c)
    ra = torch.sin((1 - t) * half) / s
    rb = torch.sin(t * half) / s
    out = ra * q0 + rb * q1
    out = torch.where(s.abs() < 0.001, 0.5 * q0 + 0.5 * q1, out)
    out = torch.where(c.abs() >= 1, q0, out)
    return out


def heading_angle(q: torch.Tensor) -> torch.Tensor:
    """phc/utils/torch_utils.py:200-212."""
    ex = torch.zeros_like(q[..., :3])
    ex[..., 0] = 1
    r = quat_rotate(q, ex)
    return torch.atan2(r[..., 1], r[..., 0])


def heading_quat(q: torch.Tensor, inverse: bool = False) -> torch.Tensor:
    """phc/utils/torch_utils.py:215-240 (calc_heading_quat / calc_heading_quat_inv)."""
    h = heading_angle(q)
    ez = torch.zeros_like(q[..., :3])
    ez[..., 2] = 1
    return quat_from_angle_axis(-h if inverse else h, ez)


# ------------------------------------------------------------------------------------------------
# MotionLib tables and queries
# ------------------------------------------------------------------------------------------------
@dataclass
class MotionTables:
    """The flat per-frame buffers MotionLibBase.load_motions builds (motion_lib_base.py:287-316)."""
    gts: torch.Tensor            # [F,24,3] global body translation
    grs: torch.Tensor            # [F,24,4] global body rotation
    lrs: torch.Tensor            # [F,24,4] local joint rotation
    gvs: torch.Tensor            # [F,24,3] global linear velocity
    gavs: torch.Tensor           # [F,24,3] global angular velocity
    dvs: torch.Tensor            # [F,23,3] dof velocity
    motion_aa: torch.Tensor      # [F,72]
    lengths: torch.Tensor        # [M] f32 seconds
    num_frames: torch.Tensor     # [M] i64
    dt: torch.Tensor             # [M] f32
    length_starts: torch.Tensor  # [M] i64 (exclusive cumsum of num_frames)
    fps: Optional[torch.Tensor] = None
    motion_bodies: Optional[torch.Tensor] = None        # [M,17]
    motion_limb_weights: Optional[torch.Tensor] = None  # [M,10]

    @property
    def num_motions(self) -> int:
        return int(self.lengths.shape[0])


def frame_blend(time: torch.Tensor, length: torch.Tensor, num_frames: torch.Tensor,
                dt: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """motion_lib_base.py:546-556 (_calc_frame_blend).  Index results are int64 and exact."""
    phase = torch.clip(time / length, 0.0, 1.0)
    time = torch.where(time < 0, torch.zeros_like(time), time)
    i0 = (phase * (num_frames - 1)).long()
    i1 = torch.min(i0 + 1, num_frames - 1)
    blend = torch.clip((time - i0 * dt) / dt, 0.0, 1.0)
    return i0, i1, blend


def motion_state(tb: MotionTables, motion_ids: torch.Tensor, motion_times: torch.Tensor,
                 offset: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """motion_lib_base.py:434-517 (get_motion_state): gather two frames, lerp / slerp."""
    i0, i1, blend = frame_blend(motion_times, tb.lengths[motion_ids], tb.num_frames[motion_ids], tb.dt[motion_ids])
    f0 = i0 + tb.length_starts[motion_ids]
    f1 = i1 + tb.length_starts[motion_ids]
    b = blend.unsqueeze(-1).unsqueeze(-1)

    pos = (1.0 - b) * tb.gts[f0] + b * tb.gts[f1]
    if offset is not None:
        pos = pos + offset[..., None, :]
    vel = (1.0 - b) * tb.gvs[f0] + b * tb.gvs[f1]
    ang_vel = (1.0 - b) * tb.gavs[f0] + b * tb.gavs[f1]
    dof_vel = (1.0 - b) * tb.dvs[f0] + b * tb.dvs[f1]
    local_rot = slerp(tb.lrs[f0], tb.lrs[f1], b)
    dof_pos = quat_to_exp_map(local_rot[:, 1:]).reshape(local_rot.shape[0], -1)  # :561-564
    rot = slerp(tb.grs[f0], tb.grs[f1], b)
    out = {
        "root_pos": pos[:, 0].clone(), "root_rot": rot[:, 0].clone(), "dof_pos": dof_pos,
        "root_vel": vel[:, 0].clone(), "root_ang_vel": ang_vel[:, 0].clone(),
        "dof_vel": dof_vel.reshape(dof_vel.shape[0], -1), "motion_aa": tb.motion_aa[f0],
        "rg_pos": pos, "rb_rot": rot, "body_vel": vel, "body_ang_vel": ang_vel,
        "frame_idx0": i0, "frame_idx1": i1, "blend": blend,
    }
    if tb.motion_bodies is not None:
        out["motion_bodies"] = tb.motion_bodies[motion_ids]
    if tb.motion_limb_weights is not None:
        out["motion_limb_weights"] = tb.motion_limb_weights[motion_ids]
    return out


def root_pos_smpl(tb: MotionTables, motion_ids: torch.Tensor, motion_times: torch.Tensor) -> torch.Tensor:
    """motion_lib_base.py:519-544 (get_root_pos_smpl)."""
    i0, i1, blend = frame_blend(motion_times, tb.lengths[motion_ids], tb.num_frames[motion_ids], tb.dt[motion_ids])
    f0 = i0 + tb.length_starts[motion_ids]
    f1 = i1 + tb.length_starts[motion_ids]
    b = blend.unsqueeze(-1).unsqueeze(-1)
    return ((1.0 - b) * tb.gts[f0] + b * tb.gts[f1])[:, 0].clone()


def sample_time_interval(tb: MotionTables, motion_ids: torch.Tensor, phase: torch.Tensor) -> torch.Tensor:
    """motion_lib_base.py:411-420 with the uniform draw `phase` supplied by the caller.

    `curr_fps = 1/30` is a python double; tensor/python-scalar on CPU divides in fp32 by fp32(1/30).
    """
    step = 1 / 30
    return ((phase * tb.lengths[motion_ids]) / step).long() * step


# ------------------------------------------------------------------------------------------------
# observation / reward / reset
# ------------------------------------------------------------------------------------------------
def self_obs_smpl_max(body_pos, body_rot, body_vel, body_ang_vel, local_root_obs: bool = True,
                      root_height_obs: bool = True) -> torch.Tensor:
    """humanoid.py:1675-1731 (compute_humanoid_observations_smpl_max), upright start, no shape obs.

    Layout: [h | R(p_j-p_0) j=1..23 | six(hinv*q_j) j=0..23 | R v_j | R w_j]  = 1+69+144+72+72.
    """
    n, nb, _ = body_pos.shape
    hinv = heading_quat(body_rot[:, 0], inverse=True).unsqueeze(1).expand(n, nb, 4)
    rel = quat_rotate(hinv, body_pos - body_pos[:, :1]).reshape(n, -1)[:, 3:]
    rot6 = quat_to_six(quat_mul(hinv, body_rot)).reshape(n, -1)
    if not local_root_obs:
        rot6 = rot6.clone()
        rot6[:, :6] = quat_to_six(body_rot[:, 0])
    vel = quat_rotate(hinv, body_vel).reshape(n, -1)
    ang = quat_rotate(hinv, body_ang_vel).reshape(n, -1)
    parts = [rel, rot6, vel, ang]
    if root_height_obs:
        parts.insert(0, body_pos[:, 0, 2:3])
    return torch.cat(parts, dim=-1)


def imitation_obs_v6(root_pos, root_rot, body_pos, body_rot, body_vel, body_ang_vel,
                     ref_pos, ref_rot, ref_vel, ref_ang_vel) -> torch.Tensor:
    """humanoid_im.py:1328-1378 (compute_imitation_observations_v6), time_steps=1, upright.

    Block-major layout over the J tracked bodies:
    [R dp | six(hinv*(qref*conj q)*h) | R dv | R dw | R (pref-root) | six(hinv*qref)] = J*(3+6+3+3+3+6).
    """
    n, nb, _ = body_pos.shape
    hinv = heading_quat(root_rot, inverse=True).unsqueeze(1).expand(n, nb, 4)
    hfwd = heading_quat(root_rot, inverse=False).unsqueeze(1).expand(n, nb, 4)
    d_pos = quat_rotate(hinv, ref_pos - body_pos)
    d_rot = quat_mul(quat_mul(hinv, quat_mul(ref_rot, quat_conj(body_rot))), hfwd)
    d_vel = quat_rotate(hinv, ref_vel - body_vel)
    d_ang = quat_rotate(hinv, ref_ang_vel - body_ang_vel)
    loc_pos = quat_rotate(hinv, ref_pos - root_pos[:, None, :])
    loc_rot = quat_to_six(quat_mul(hinv, ref_rot))
    blocks = [d_pos, quat_to_six(d_rot), d_vel, d_ang, loc_pos, loc_rot]
    return torch.cat([x.reshape(n, -1) for x in blocks], dim=-1)


def imitation_obs_v7(root_pos, root_rot, body_pos, body_vel, ref_pos, ref_vel) -> torch.Tensor:
    """humanoid_im.py:1381-1413 (compute_imitation_observations_v7): [R dp | R dv | R (pref-root)]."""
    n, nb, _ = body_pos.shape
    hinv = heading_quat(root_rot, inverse=True).unsqueeze(1).expand(n, nb, 4)
    blocks = [quat_rotate(hinv, ref_pos - body_pos), quat_rotate(hinv, ref_vel - body_vel),
              quat_rotate(hinv, ref_pos - root_pos[:, None, :])]
    return torch.cat([x.reshape(n, -1) for x in blocks], dim=-1)


def remove_base_rot(q: torch.Tensor) -> torch.Tensor:
    """humanoid.py:1617-1620: q (x) conj([.5, .5, .5, .5]) -- the SMPL rest orientation of a non-upright start."""
    base = quat_conj(torch.tensor([[0.5, 0.5, 0.5, 0.5]], dtype=q.dtype)).expand(q.shape[0], 4)
    return quat_mul(q, base)


TASK_OBS_VERSIONS = (1, 2, 3, 6, 7, 8, 9)


def imitation_obs(version: int, root_pos, root_rot, body_pos, body_rot, body_vel, body_ang_vel, ref_pos, ref_rot, ref_vel, ref_ang_vel,
                  time_steps: int = 1, upright: bool = True, dof_pos=None, ref_dof_pos=None) -> torch.Tensor:
    """Every `compute_imitation_observations*` variant `_compute_task_obs` dispatches on (humanoid_im.py:757-833) for J tracked bodies
    and `time_steps` future samples (fut_tracks).  body_* [B, J, .] are the SUBSET rows; ref_* [B * time_steps, J, .] in the reference's
    `repeat_interleave(time_steps)` order (row b * T + t).

      1  :1222-1258  [dp | six(drot) | dv | dw]                                   flat over (t, j)
      2  :1261-1301  version 1 + (ref_dof_pos - dof_pos) of the tracked joints    (time_steps = 1)
      3  :1304-1326  [dp | six(drot)]
      6  :1328-1378  per t: [dp_t | six(drot_t) | dv_t | dw_t | R(pref_t - root) | six(hinv qref_t)]
      7  :1381-1413  per t: [dp_t | dv_t | R(pref_t - root)]
      8  :1415-1479  diffs of sample 0 + [R(pref - root) | six(hinv qref) | R vref | R wref]   (time_steps = 1 branch, :1472-1476)
      9  :1482-1540  per t: [dp_t | six(drot_t) | R(v_ref_root - v_root) | R(w_ref_root - w_root) | R(pref_t - root) | six(hinv qref_t)]
    """
    B, J, _ = body_pos.shape
    T = time_steps
    if not upright:
        root_rot = remove_base_rot(root_rot)
    hinv = heading_quat(root_rot, inverse=True)[:, None, None, :].expand(B, T, J, 4)
    hfwd = heading_quat(root_rot, inverse=False)[:, None, None, :].expand(B, T, J, 4)
    rp, rr, rv, rw = ref_pos.view(B, T, J, 3), ref_rot.view(B, T, J, 4), ref_vel.view(B, T, J, 3), ref_ang_vel.view(B, T, J, 3)
    bp, br, bv, bw = body_pos[:, None], body_rot[:, None].expand(B, T, J, 4), body_vel[:, None], body_ang_vel[:, None]
    d_pos = quat_rotate(hinv, rp - bp)
    d_rot6 = quat_to_six(quat_mul(quat_mul(hinv, quat_mul(rr, quat_conj(br))), hfwd))
    d_vel = quat_rotate(hinv, rv - bv)
    d_ang = quat_rotate(hinv, rw - bw)
    loc_pos = quat_rotate(hinv, rp - root_pos[:, None, None, :])
    loc_rot6 = quat_to_six(quat_mul(hinv, rr))
    flat = lambda x: x.reshape(B, -1)
    per_t = lambda *xs: torch.cat([x.reshape(B, T, -1) for x in xs], dim=-1).reshape(B, -1)
    if version == 1:
        return torch.cat([flat(d_pos), flat(d_rot6), flat(d_vel), flat(d_ang)], dim=-1)
    if version == 2:
        assert T == 1
        return torch.cat([flat(d_pos), flat(d_rot6), flat(d_vel), flat(d_ang), flat(ref_dof_pos.view(B, -1) - dof_pos.view(B, -1))], dim=-1)
    if version == 3:
        return torch.cat([flat(d_pos), flat(d_rot6)], dim=-1)
    if version == 6:
        return per_t(d_pos, d_rot6, d_vel, d_ang, loc_pos, loc_rot6)
    if version == 7:
        return per_t(d_pos, d_vel, loc_pos)
    if version == 8:
        assert T == 1
        loc_vel, loc_ang = quat_rotate(hinv, rv), quat_rotate(hinv, rw)
        return torch.cat([flat(d_pos), flat(d_rot6), flat(d_vel), flat(d_ang), flat(loc_pos), flat(loc_rot6), flat(loc_vel), flat(loc_ang)], dim=-1)
    if version == 9:
        h1 = hinv[:, :, 0]
        d_rv = quat_rotate(h1, rv[:, :, 0] - body_vel[:, None, 0])
        d_rw = quat_rotate(h1, rw[:, :, 0] - body_ang_vel[:, None, 0])
        return per_t(d_pos, d_rot6, d_rv, d_rw, loc_pos, loc_rot6)
    raise ValueError(f"obs version {version}")


REWARD_SPECS = {"k_pos": 100.0, "k_rot": 10.0, "k_vel": 0.1, "k_ang_vel": 0.1,
                "w_pos": 0.5, "w_rot": 0.3, "w_vel": 0.1, "w_ang_vel": 0.1}  # humanoid_im.py:55


def imitation_reward(body_pos, body_rot, body_vel, body_ang_vel, ref_pos, ref_rot, ref_vel, ref_ang_vel,
                     specs: Dict[str, float] = REWARD_SPECS) -> Tuple[torch.Tensor, torch.Tensor]:
    """humanoid_im.py:1543-1574 (compute_imitation_reward)."""
    e_pos = ((ref_pos - body_pos) ** 2).mean(dim=-1).mean(dim=-1)
    ang = quat_to_angle_axis(quat_mul(ref_rot, quat_conj(body_rot)))[0]
    e_rot = (ang ** 2).mean(dim=-1)
    e_vel = ((ref_vel - body_vel) ** 2).mean(dim=-1).mean(dim=-1)
    e_ang = ((ref_ang_vel - body_ang_vel) ** 2).mean(dim=-1).mean(dim=-1)
    r_pos = torch.exp(-specs["k_pos"] * e_pos)
    r_rot = torch.exp(-specs["k_rot"] * e_rot)
    r_vel = torch.exp(-specs["k_vel"] * e_vel)
    r_ang = torch.exp(-specs["k_ang_vel"] * e_ang)
    rew = specs["w_pos"] * r_pos + specs["w_rot"] * r_rot + specs["w_vel"] * r_vel + specs["w_ang_vel"] * r_ang
    return rew, torch.stack([r_pos, r_rot, r_vel, r_ang], dim=-1)


def im_reset(reset_buf, progress_buf, body_pos_subset, ref_pos_subset, pass_time, termination_distance,
             enable_early_termination: bool = True, use_mean: bool = False,
             disable_collision: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """humanoid_im.py:1600-1628 (compute_humanoid_im_reset). int64 outputs."""
    terminated = torch.zeros_like(reset_buf)
    if enable_early_termination:
        dist = torch.norm(body_pos_subset - ref_pos_subset, dim=-1)
        if use_mean:
            fallen = torch.any(dist.mean(dim=-1, keepdim=True) > termination_distance[0], dim=-1)
        else:
            fallen = torch.any(dist > termination_distance, dim=-1)
        fallen = fallen & (progress_buf > 1)
        if disable_collision:
            fallen = torch.zeros_like(fallen)
        terminated = torch.where(fallen, torch.ones_like(reset_buf), terminated)
    reset = torch.where(pass_time, torch.ones_like(reset_buf), terminated)
    return reset, terminated


def amp_dof_subset() -> torch.Tensor:
    keep = [k for k in range(NUM_DOF) if (k // 3) not in AMP_DROPPED_JOINTS]
    return torch.tensor(keep, dtype=torch.long)


def amp_obs_smpl(root_pos, root_rot, root_vel, root_ang_vel, dof_pos, dof_vel, key_body_pos,
                 dof_subset: Optional[torch.Tensor] = None, local_root_obs: bool = True,
                 root_height_obs: bool = True) -> torch.Tensor:
    """humanoid_amp.py:924-969 (build_amp_observations_smpl), upright, no shape/limb obs.

    [h | six(hinv*q0) | R v0 | R w0 | six(exp_map_to_quat(dof)) per kept joint | dof_vel kept | R (key-p0)].
    """
    n = root_pos.shape[0]
    hinv = heading_quat(root_rot, inverse=True)
    root6 = quat_to_six(quat_mul(hinv, root_rot) if local_root_obs else root_rot)
    lv = quat_rotate(hinv, root_vel)
    la = quat_rotate(hinv, root_ang_vel)
    nk = key_body_pos.shape[1]
    key = quat_rotate(hinv.unsqueeze(1).expand(n, nk, 4), key_body_pos - root_pos.unsqueeze(1)).reshape(n, -1)
    if dof_subset is not None:
        dof_pos = dof_pos[:, dof_subset]
        dof_vel = dof_vel[:, dof_subset]
    dof6 = quat_to_six(exp_map_to_quat(dof_pos.reshape(-1, 3))).reshape(n, -1)  # humanoid.py:1436-1446
    parts = [root6, lv, la, dof6, dof_vel, key]
    if root_height_obs:
        parts.insert(0, root_pos[:, 2:3])
    return torch.cat(parts, dim=-1)


# ------------------------------------------------------------------------------------------------
# one HumanoidIm post-physics step (reward -> reset -> observation), SURVEY Appendix A.9
# ------------------------------------------------------------------------------------------------
@dataclass
class ImStepConfig:
    dt: float = STEP_DT
    power_reward: bool = True            # env_im.yaml:23
    power_coefficient: float = 0.0005    # humanoid_im.py:91
    max_episode_length: int = 300        # env_im.yaml:8
    enable_early_termination: bool = True
    termination_distance: float = 0.25   # env_im.yaml:41
    cycle_motion: bool = False           # env_im.yaml:17
    use_mean_reset: bool = False         # flags.im_eval and not strict_eval
    reset_body_ids: Tuple[int, ...] = RESET_BODY_IDS
    reward_specs: Dict[str, float] = field(default_factory=lambda: dict(REWARD_SPECS))


def im_motion_times(progress_buf, start_times, start_offset, dt: float, plus_one: bool) -> torch.Tensor:
    """humanoid_im.py:732 / :859 / :1120 -- three separate fp32 ops on an int64 progress counter."""
    p = progress_buf + 1 if plus_one else progress_buf
    return p * dt + start_times + start_offset


def humanoid_im_step(tb: MotionTables, cfg: ImStepConfig, body_state: torch.Tensor, dof_vel: torch.Tensor,
                     dof_force: torch.Tensor, progress_buf: torch.Tensor, motion_ids: torch.Tensor,
                     start_times: torch.Tensor, start_offset: torch.Tensor, global_offset: torch.Tensor,
                     cycle_counter: torch.Tensor, reset_buf: torch.Tensor,
                     recovery_counter: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """HumanoidIm.post_physics_step compute, non-cycling branch, after `progress_buf += 1`.
    With `recovery_counter` the HumanoidImGetup override of `_compute_reset` (humanoid_im_getup.py:203-210) is applied:
    recovering envs are never reset and their progress counter is pulled back by one BEFORE the observation is computed
    (out["progress_buf"] is the counter after the step).

    humanoid_im.py:853-919 (_compute_reward), :1119-1192 (_compute_reset), :677-851
    (_compute_observations / _compute_task_obs, obs_v 6), humanoid.py:1137-1213 (_compute_humanoid_obs).
    `body_state` is the Isaac Gym rigid-body-state view [N,24,13] = pos, quat xyzw, linvel, angvel.
    """
    pos, rot, vel, ang = body_state[..., 0:3], body_state[..., 3:7], body_state[..., 7:10], body_state[..., 10:13]
    out: Dict[str, torch.Tensor] = {}

    # reward at t = progress*dt + start + offset
    t_rew = im_motion_times(progress_buf, start_times, start_offset, cfg.dt, plus_one=False)
    ref = motion_state(tb, motion_ids, t_rew, global_offset)
    rew, raw = imitation_reward(pos, rot, vel, ang, ref["rg_pos"], ref["rb_rot"], ref["body_vel"],
                                ref["body_ang_vel"], cfg.reward_specs)
    if cfg.power_reward:
        power = torch.abs(torch.multiply(dof_force, dof_vel)).sum(dim=-1)
        p_rew = -cfg.power_coefficient * power
        p_rew = torch.where(progress_buf <= 3, torch.zeros_like(p_rew), p_rew)
        rew = rew + p_rew
        raw = torch.cat([raw, p_rew[:, None]], dim=-1)
    out["rew_buf"], out["reward_raw"] = rew, raw

    # reset at the same t (the reference reuses the cached query, humanoid_im.py:950-964)
    if cfg.cycle_motion:
        pass_time = progress_buf >= cfg.max_episode_length - 1
    else:
        pass_time = t_rew >= tb.lengths[motion_ids]
    rb = torch.tensor(cfg.reset_body_ids, dtype=torch.long)
    term_dist = torch.full((1, NUM_BODIES), cfg.termination_distance, dtype=F32)[..., rb]
    reset, terminated = im_reset(reset_buf, progress_buf, pos[:, rb], ref["rg_pos"][:, rb], pass_time, term_dist,
                                 cfg.enable_early_termination, cfg.use_mean_reset)
    recovering = torch.logical_and(~pass_time, cycle_counter > 0)
    reset = torch.where(recovering, torch.zeros_like(reset), reset)
    terminated = torch.where(recovering, torch.zeros_like(terminated), terminated)
    if recovery_counter is not None:                      # humanoid_im_getup.py:206-209
        is_rec = recovery_counter > 0
        reset = torch.where(is_rec, torch.zeros_like(reset), reset)
        terminated = torch.where(is_rec, torch.zeros_like(terminated), terminated)
        progress_buf = torch.where(is_rec, progress_buf - 1, progress_buf)
        out["progress_buf"] = progress_buf
    out["reset_buf"], out["terminate_buf"] = reset, terminated
    out["frame_idx_rew"] = torch.stack([ref["frame_idx0"], ref["frame_idx1"]], dim=-1)

    # observation at t + dt
    t_obs = im_motion_times(progress_buf, start_times, start_offset, cfg.dt, plus_one=True)
    nxt = motion_state(tb, motion_ids, t_obs, global_offset)
    self_obs = self_obs_smpl_max(pos, rot, vel, ang)
    task_obs = imitation_obs_v6(pos[:, 0], rot[:, 0], pos, rot, vel, ang, nxt["rg_pos"], nxt["rb_rot"],
                                nxt["body_vel"], nxt["body_ang_vel"])
    out["obs_buf"] = torch.cat([self_obs, task_obs], dim=-1)
    out["ref_body_pos"], out["ref_body_rot"], out["ref_body_vel"] = nxt["rg_pos"], nxt["rb_rot"], nxt["body_vel"]
    out["ref_dof_pos"] = nxt["dof_pos"]
    out["frame_idx_obs"] = torch.stack([nxt["frame_idx0"], nxt["frame_idx1"]], dim=-1)
    return out


def amp_obs_step(amp_obs_buf: torch.Tensor, body_state: torch.Tensor, dof_pos: torch.Tensor,
                 dof_vel: torch.Tensor) -> torch.Tensor:
    """humanoid_amp.py:622-630 + 632-667: hist[1:] <- buf[:-1]; buf[0] <- current AMP obs. Returns new buffer."""
    cur = amp_obs_smpl(body_state[:, 0, 0:3], body_state[:, 0, 3:7], body_state[:, 0, 7:10], body_state[:, 0, 10:13],
                       dof_pos, dof_vel, body_state[:, list(KEY_BODY_IDS), 0:3], amp_dof_subset())
    return torch.cat([cur.unsqueeze(1), amp_obs_buf[:, :-1]], dim=1)


def reset_envs(tb: MotionTables, cfg: ImStepConfig, st: Dict[str, torch.Tensor], env_ids: torch.Tensor, phase: torch.Tensor,
               num_amp_steps: int = 10) -> Dict[str, torch.Tensor]:
    """The reference's per-step env reset for the envs in `env_ids` (ascending, what `nonzero` returns), restated as one function
    over a dict of buffers (all updated copies are returned; `phase[e]` is the uniform draw of env e):

      Humanoid._reset_envs (humanoid.py:574-587)
        -> HumanoidIm._reset_ref_state_init (humanoid_im.py:921-948): start offset, global offset, cycle counter <- 0
        -> HumanoidAMP._reset_ref_state_init (humanoid_amp.py:468-488) / _sample_ref_state (humanoid_im.py:966-989):
           start time = sample_time_interval (motion_lib_base.py:411-420), get_motion_state with the (zeroed) global offset
        -> _set_env_state (humanoid_amp.py:565-597): root 13, dof pos / vel, rigid bodies (kept after the refresh, :604-614)
        -> _reset_env_tensors (humanoid.py:589-609): progress / reset / terminate / contact forces <- 0
        -> _compute_observations(env_ids) (humanoid_im.py:677-706)
      HumanoidAMP._init_amp_obs (humanoid_amp.py:519-563): current AMP observation from the state just set, history rows from the
      reference motion at t0 - dt*(k), k = 1 .. num_amp_steps-1, WITHOUT offset.

    st keys: motion_ids, start_times, start_offset, global_offset [N,3], cycle_counter, progress_buf, reset_buf, terminate_buf,
    root_states [N,13], dof_pos [N,69], dof_vel [N,69], body_state [N,24,13], contact_forces [N,24,3], amp_obs_buf [N,steps,196],
    obs_buf [N,934], dof_force [N,69]."""
    o = {k: v.clone() for k, v in st.items()}
    ids = env_ids.long()
    n = ids.shape[0]
    if n == 0:
        return o
    mids = o["motion_ids"][ids]
    o["start_offset"][ids] = 0
    o["global_offset"][ids] = 0
    o["cycle_counter"][ids] = 0
    t0 = sample_time_interval(tb, mids, phase[ids])
    ms = motion_state(tb, mids, t0, o["global_offset"][ids])
    o["root_states"][ids] = torch.cat([ms["root_pos"], ms["root_rot"], ms["root_vel"], ms["root_ang_vel"]], dim=-1)
    o["dof_pos"][ids] = ms["dof_pos"]
    o["dof_vel"][ids] = ms["dof_vel"]
    o["body_state"][ids] = torch.cat([ms["rg_pos"], ms["rb_rot"], ms["body_vel"], ms["body_ang_vel"]], dim=-1)
    o["start_times"][ids] = t0
    o["progress_buf"][ids] = 0
    o["reset_buf"][ids] = 0
    o["terminate_buf"][ids] = 0
    o["contact_forces"][ids] = 0
    # _compute_observations(env_ids): progress 0 -> observation query at dt + t0
    sub = humanoid_im_step(tb, cfg, o["body_state"][ids], o["dof_vel"][ids], o["dof_force"][ids], o["progress_buf"][ids], mids, t0,
                           o["start_offset"][ids], o["global_offset"][ids], o["cycle_counter"][ids], o["reset_buf"][ids])
    o["obs_buf"][ids] = sub["obs_buf"]
    # _init_amp_obs: slot 0 from the simulator tensors just written, slots 1.. from the reference motion (no offset)
    bs = o["body_state"][ids]
    cur = amp_obs_smpl(bs[:, 0, 0:3], bs[:, 0, 3:7], bs[:, 0, 7:10], bs[:, 0, 10:13], o["dof_pos"][ids], o["dof_vel"][ids],
                       bs[:, list(KEY_BODY_IDS), 0:3], amp_dof_subset())
    rows = [cur]
    for k in range(1, num_amp_steps):
        t_k = t0 + (-cfg.dt) * k
        h = motion_state(tb, mids, t_k)
        rows.append(amp_obs_smpl(h["root_pos"], h["root_rot"], h["root_vel"], h["root_ang_vel"], h["dof_pos"], h["dof_vel"],
                                 h["rg_pos"][:, list(KEY_BODY_IDS)], amp_dof_subset()))
    o["amp_obs_buf"][ids] = torch.stack(rows, dim=1)
    return o


# ------------------------------------------------------------------------------------------------
# rollout post-processing: GAE, returns, advantage normalisation
# ------------------------------------------------------------------------------------------------
def discount_values(fdones, values, rewards, next_values, gamma: float = 0.99, tau: float = 0.95) -> torch.Tensor:
    """common_agent.py:493-505. Shapes [T,N] dones, [T,N,1] others."""
    last = 0
    advs = torch.zeros_like(rewards)
    for t in reversed(range(rewards.shape[0])):
        not_done = (1.0 - fdones[t]).unsqueeze(1)
        delta = rewards[t] + gamma * next_values[t] - values[t]
        last = delta + gamma * tau * not_done * last
        advs[t] = last
    return advs


def swap_and_flatten01(x: torch.Tensor) -> torch.Tensor:
    """rl_games a2c_common.swap_and_flatten01 [3P-memory]: [T,N,...] -> env-major [N*T,...]."""
    return x.transpose(0, 1).reshape(x.shape[0] * x.shape[1], *x.shape[2:])


def normalized_advantages(returns: torch.Tensor, values: torch.Tensor) -> torch.Tensor:
    """common_agent.py:589-599 (_calc_advs, normalize_advantage=True)."""
    adv = torch.sum(returns - values, dim=1)
    return (adv - adv.mean()) / (adv.std() + 1e-8)


class RunningMeanStd:
    """phc/utils/running_mean_std.py:9-109 (per-feature, fp64 statistics, clamp +-5)."""

    def __init__(self, size: int, epsilon: float = 1e-5):
        self.mean = torch.zeros(size, dtype=torch.float64)
        self.var = torch.ones(size, dtype=torch.float64)
        self.count = torch.ones((), dtype=torch.float64)
        self.eps = epsilon

    def update(self, x: torch.Tensor) -> None:
        mean, var, n = x.mean(0), x.var(0), x.shape[0]
        delta = mean - self.mean
        tot = self.count + n
        new_mean = self.mean + delta * n / tot
        m2 = self.var * self.count + var * n + delta ** 2 * self.count * n / tot
        self.mean, self.var, self.count = new_mean, m2 / tot, tot

    def normalize(self, x: torch.Tensor, unnorm: bool = False) -> torch.Tensor:
        if unnorm:
            y = torch.clamp(x, min=-5.0, max=5.0)
            return torch.sqrt(self.var.float() + self.eps) * y + self.mean.float()
        y = (x - self.mean.float()) / torch.sqrt(self.var.float() + self.eps)
        return torch.clamp(y, min=-5.0, max=5.0)


# ------------------------------------------------------------------------------------------------
# networks and losses
# ------------------------------------------------------------------------------------------------
def mlp_forward(x: torch.Tensor, weights, biases, activation: str = "relu", last_linear: bool = False) -> torch.Tensor:
    """network_builder.py:105-124 style Linear+activation stack (fp32)."""
    act = {"relu": torch.relu, "silu": torch.nn.functional.silu}[activation]
    for i, (w, b) in enumerate(zip(weights, biases)):
        x = torch.nn.functional.linear(x, w, b)
        if not (last_linear and i == len(weights) - 1):
            x = act(x)
    return x


def gaussian_neglogp(x, mu, sigma, logstd) -> torch.Tensor:
    """rl_games ModelA2CContinuousLogStd.neglogp [3P-memory]."""
    return 0.5 * (((x - mu) / sigma) ** 2).sum(dim=-1) + 0.5 * math.log(2.0 * math.pi) * x.shape[-1] + logstd.sum(dim=-1)


def actor_loss(old_neglogp, neglogp, advantage, e_clip: float = 0.2) -> torch.Tensor:
    """common_agent.py:564-574."""
    ratio = torch.exp(old_neglogp - neglogp)
    return torch.max(-advantage * ratio, -advantage * torch.clamp(ratio, 1.0 - e_clip, 1.0 + e_clip))


def critic_loss(values, returns) -> torch.Tensor:
    """common_agent.py:576-587 with clip_value False (im.yaml:75)."""
    return (returns - values) ** 2


def bound_loss(mu, soft_bound: float = 1.0) -> torch.Tensor:
    """common_agent.py:512-520."""
    hi = torch.clamp_min(mu - soft_bound, 0.0) ** 2
    lo = torch.clamp_max(mu + soft_bound, 0.0) ** 2
    return (lo + hi).sum(dim=-1)


def policy_kl(mu0, sigma0, mu1, sigma1) -> torch.Tensor:
    """rl_games torch_ext.policy_kl, reduce=True [3P-memory]."""
    c1 = torch.log(sigma1 / sigma0 + 1e-5)
    c2 = (sigma0 ** 2 + (mu1 - mu0) ** 2) / (2.0 * (sigma1 ** 2 + 1e-5))
    return (c1 + c2 - 0.5).sum(dim=-1).mean()


def disc_reward(logits, scale: float = 2.0) -> torch.Tensor:
    """amp_agent.py:1027-1041 (no disc-reward normaliser)."""
    prob = 1 / (1 + torch.exp(-logits))
    return -torch.log(torch.maximum(1 - prob, torch.tensor(0.0001))) * scale


def kl_multi(mu_q, logvar_q, mu_p, logvar_p) -> torch.Tensor:
    """phc/learning/loss_functions.py:3-11: KL(q||p) of diagonal Gaussians, summed over the latent."""
    per_dim = 0.5 * (logvar_p - logvar_q + logvar_q.exp() / logvar_p.exp()
                     + (mu_q - mu_p).pow(2) / logvar_p.exp() - 1)
    return per_dim.sum(-1)


def ppo_total_loss(mu, value, old_neglogp, advantage, returns, actions, logstd, e_clip=0.2,
                   critic_coef=5.0, bounds_coef=10.0) -> Dict[str, torch.Tensor]:
    """amp_agent.py:691-710 without the discriminator term (entropy_coef 0)."""
    sigma = torch.exp(logstd).expand_as(mu)
    neglogp = gaussian_neglogp(actions, mu, sigma, logstd.expand_as(mu))
    a = actor_loss(old_neglogp, neglogp, advantage, e_clip).mean()
    c = critic_loss(value, returns).mean()
    b = bound_loss(mu).mean()
    return {"a_loss": a, "c_loss": c, "b_loss": b, "loss": a + critic_coef * c + bounds_coef * b, "neglogp": neglogp}


def disc_loss(disc_mlp, amp_agent, amp_replay, amp_demo, logit_weight, all_weights, logit_reg: float = 0.01,
              grad_penalty: float = 5.0, weight_decay: float = 0.0001) -> Dict[str, torch.Tensor]:
    """amp_agent.py:895-952 (_disc_loss) incl. the eval_disc calls of amp_models.py:33-41.

    `disc_mlp` maps (already normalised) AMP observations to logits; `logit_weight` is `_disc_logits.weight`,
    `all_weights` the weights of every discriminator Linear layer (get_disc_weights, amp_network_builder.py:221-228)."""
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    demo = amp_demo.detach().clone().requires_grad_(True)
    agent_logit = torch.cat([disc_mlp(amp_agent), disc_mlp(amp_replay)], dim=0)
    demo_logit = disc_mlp(demo)
    loss = 0.5 * (bce(agent_logit, torch.zeros_like(agent_logit)) + bce(demo_logit, torch.ones_like(demo_logit)))
    logit_loss = torch.sum(torch.square(torch.flatten(logit_weight)))
    loss = loss + logit_reg * logit_loss
    grad = torch.autograd.grad(demo_logit, demo, grad_outputs=torch.ones_like(demo_logit), create_graph=True, retain_graph=True,
                               only_inputs=True)[0]
    gp = torch.mean(torch.sum(torch.square(grad), dim=-1))
    loss = loss + grad_penalty * gp
    if weight_decay != 0:
        wd = torch.sum(torch.square(torch.cat([torch.flatten(w) for w in all_weights], dim=-1)))
        loss = loss + weight_decay * wd
    return {"disc_loss": loss, "disc_grad_penalty": gp.detach(), "disc_logit_loss": logit_loss.detach(),
            "disc_agent_acc": (agent_logit < 0).float().mean(), "disc_demo_acc": (demo_logit > 0).float().mean()}


# ------------------------------------------------------------------------------------------------
# PULSE VAE distillation (SURVEY K17-K19), Z-task decode (K20), reach task (K21), PD targets (K22)
# ------------------------------------------------------------------------------------------------
@dataclass
class VaeNets:
    """Weights of `AMPZBuilder.Network` (amp_network_z_builder.py:469-557) as (weights, biases) lists, reference layout.

    enc: z_mlp = [Linear+SiLU]*len(task units) + Linear(units[-1], 5*E)  (:492-497);  enc_mu / enc_logvar: Linear(5E, E) (:510-512)
    prior: z_prior = [Linear+SiLU]*len(task units) (:517);  prior_mu / prior_logvar: Linear(units[-1], E) (:518-519)
    dec: actor_mlp = [Linear+SiLU]*len(mlp units) on [self_obs, z], then `mu` Linear (network_builder.py:246,261)
    critic_z: critic_z_mlp (same shape as z_mlp but E outputs), critic: critic_mlp on [self_obs, critic_z] + `value`."""
    enc: Tuple[list, list]
    enc_mu: Tuple[torch.Tensor, torch.Tensor]
    enc_logvar: Tuple[torch.Tensor, torch.Tensor]
    prior: Tuple[list, list]
    prior_mu: Tuple[torch.Tensor, torch.Tensor]
    prior_logvar: Tuple[torch.Tensor, torch.Tensor]
    dec: Tuple[list, list]
    critic_z: Optional[Tuple[list, list]] = None
    critic: Optional[Tuple[list, list]] = None
    self_obs_size: int = SELF_OBS
    clamp_lo: float = -5.0          # use_vae_clamped_prior (:86-87, :234-235)
    clamp_hi: float = 2.0           # vae_var_clamp_max, env_im_vae.yaml:27

    @staticmethod
    def from_state_dict(sd: Dict[str, torch.Tensor], self_obs_size: int, prefix: str = "", clamp_hi: float = 2.0) -> "VaeNets":
        def seq(name):
            idx = sorted({int(k[len(prefix + name) + 1:].split(".")[0]) for k in sd if k.startswith(prefix + name + ".")})
            return ([torch.as_tensor(sd[f"{prefix}{name}.{i}.weight"]) for i in idx], [torch.as_tensor(sd[f"{prefix}{name}.{i}.bias"]) for i in idx])

        def lin(name):
            return torch.as_tensor(sd[f"{prefix}{name}.weight"]), torch.as_tensor(sd[f"{prefix}{name}.bias"])

        dec = seq("actor_mlp")
        dec[0].append(lin("mu")[0]); dec[1].append(lin("mu")[1])
        crit = None
        if f"{prefix}critic_mlp.0.weight" in sd:
            crit = seq("critic_mlp")
            crit[0].append(lin("value")[0]); crit[1].append(lin("value")[1])
        return VaeNets(enc=seq("z_mlp"), enc_mu=lin("z_mu"), enc_logvar=lin("z_logvar"), prior=seq("z_prior"), prior_mu=lin("z_prior_mu"),
                       prior_logvar=lin("z_prior_logvar"), dec=dec, critic_z=seq("critic_z_mlp") if f"{prefix}critic_z_mlp.0.weight" in sd else None,
                       critic=crit, self_obs_size=self_obs_size, clamp_hi=clamp_hi)


def vae_encode(nets: VaeNets, obs: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """z_mlp -> z_mu / clamped z_logvar (amp_network_z_builder.py:432, :82-87)."""
    h = mlp_forward(obs, *nets.enc, activation="silu", last_linear=True)
    mu = torch.nn.functional.linear(h, *nets.enc_mu)
    lv = torch.clamp(torch.nn.functional.linear(h, *nets.enc_logvar), min=nets.clamp_lo, max=nets.clamp_hi)
    return mu, lv


def vae_prior(nets: VaeNets, obs: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """compute_prior (amp_network_z_builder.py:226-241), use_vae_prior + use_vae_clamped_prior."""
    h = mlp_forward(obs[:, :nets.self_obs_size], *nets.prior, activation="silu")
    mu = torch.nn.functional.linear(h, *nets.prior_mu)
    lv = torch.clamp(torch.nn.functional.linear(h, *nets.prior_logvar), min=nets.clamp_lo, max=nets.clamp_hi)
    return mu, lv


def vae_decode(nets: VaeNets, self_obs: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """actor_mlp([self_obs, z]) -> mu (amp_network_z_builder.py:445-462)."""
    return mlp_forward(torch.cat([self_obs, z], dim=-1), *nets.dec, activation="silu", last_linear=True)


def vae_eval_actor(nets: VaeNets, obs: torch.Tensor, noise: torch.Tensor) -> Dict[str, torch.Tensor]:
    """eval_actor(return_extra=True) with the reparameterisation noise given (amp_network_z_builder.py:341-467, :89-90, :243-246)."""
    mu, lv = vae_encode(nets, obs)
    z = mu + torch.exp(0.5 * lv) * noise
    return {"pred_action": vae_decode(nets, obs[:, :nets.self_obs_size], z), "vae_mu": mu, "vae_log_var": lv, "z": z}


def vae_eval_critic(nets: VaeNets, obs: torch.Tensor) -> torch.Tensor:
    """eval_critic, non-RNN branch for z_type 'vae' (amp_network_z_builder.py:325-339)."""
    cz = mlp_forward(obs, *nets.critic_z, activation="silu", last_linear=True)
    return mlp_forward(torch.cat([obs[:, :nets.self_obs_size], cz], dim=-1), *nets.critic, activation="silu", last_linear=True)


def vae_kin_loss(nets: VaeNets, obs: torch.Tensor, noise: torch.Tensor, gt_action: torch.Tensor, progress: torch.Tensor, horizon: int,
                 kld_coef: float = 0.01, ar1_coef: float = 0.005, use_ar1: bool = True, use_regu: bool = False, phi: float = 0.99) -> Dict[str, torch.Tensor]:
    """AMPAgent._optimize_kin, z_type 'vae' + use_vae_prior (amp_agent.py:771-849).  rows are env-major [B/horizon, horizon]."""
    out = vae_eval_actor(nets, obs, noise)
    action_loss = torch.norm(out["pred_action"] - gt_action, dim=-1).mean()                       # :782
    pm, plv = vae_prior(nets, obs)
    kld = kl_multi(out["vae_mu"], out["vae_log_var"], pm, plv).mean()                             # :786-787
    ar1 = torch.zeros(())
    if use_ar1:                                                                                   # :792-808
        B = obs.shape[0]
        tz = out["vae_mu"].view(B // horizon, horizon, -1)
        err = tz[:, 1:] - tz[:, :-1] * phi
        idx = progress.view(B // horizon, horizon, -1)
        not_consec = ((idx[:, 1:] - idx[:, :-1]) != 1).view(-1)
        starters = ((idx <= 2)[:, 1:] + (idx <= 2)[:, :-1]).view(-1)
        keep = (~(not_consec | starters)).to(err.dtype).view(-1, 1)
        ar1 = torch.norm(err.reshape(-1, err.shape[-1]) * keep, dim=-1).mean()
    regu = torch.zeros(())
    if use_regu:                                                                                  # :810-814
        regu = ((pm ** 2).mean() + (out["vae_mu"] ** 2).mean()) * 0.001 + ((plv ** 2).mean() + (out["vae_log_var"] ** 2).mean()) * 0.001
    loss = action_loss + kld * kld_coef + ar1 * ar1_coef + regu * 0.005                           # :816
    return {"kin_loss": loss, "kin_action_loss": action_loss, "kin_KLD": kld, "kin_ar1": ar1, "kin_prior_regu": regu, **out,
            "prior_mu": pm, "prior_log_var": plv}


def kld_anneal(epoch: int, kld_min: float = 0.001, start: int = 2500, end: int = 5000, base: float = 0.01) -> float:
    """amp_agent.py:827-833: the coefficient used from `epoch` on (unchanged before `start`)."""
    return (base - kld_min) * max((end - epoch) / (end - start), 0) + kld_min


def teacher_action(raw_obs, mean, var, pnn_cols, composer, self_obs_size: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """HumanoidImDistill.step (humanoid_im_distill.py:167-198): normalise with the TEACHER's statistics, clamp +-5, three frozen
    ReLU columns (PNN without lateral links, pnn.py:127-131) and the composer MLP as rebuilt by load_mcp_mlp (activation after
    EVERY Linear including the last, network_loader.py:37-39); action = sum_k w_k a_k.
    pnn_cols: list of (weights, biases); composer: (weights, biases)."""
    so = (raw_obs[:, :self_obs_size] - mean.float()[:self_obs_size]) / torch.sqrt(var.float()[:self_obs_size] + 1e-05)
    to = (raw_obs[:, self_obs_size:] - mean.float()[self_obs_size:]) / torch.sqrt(var.float()[self_obs_size:] + 1e-05)
    x = torch.clamp(torch.cat([so, to], dim=-1), min=-5.0, max=5.0)
    acts = torch.stack([mlp_forward(x, w, b, activation="relu", last_linear=True) for w, b in pnn_cols], dim=1)
    wts = mlp_forward(x, *composer, activation="silu", last_linear=False)
    return torch.sum(wts[:, :, None] * acts, dim=1), wts


def z_decode_actions(nets: VaeNets, raw_obs: torch.Tensor, mean, var, action_z: torch.Tensor) -> torch.Tensor:
    """HumanoidZ.compute_z_actions, 'vae' + use_vae_prior (humanoid_z.py:81-155): the prior sees the UNCLAMPED normalised self
    observation, the decoder the clamped one; z = prior_mu + action_z (project_to_norm(.., 'none') is the identity)."""
    S = nets.self_obs_size
    so = (raw_obs[:, :S] - mean.float()[:S]) / torch.sqrt(var.float()[:S] + 1e-05)
    pm = torch.nn.functional.linear(mlp_forward(so, *nets.prior, activation="silu"), *nets.prior_mu)
    return vae_decode(nets, torch.clamp(so, min=-5.0, max=5.0), pm + action_z)


def reach_obs(root_states: torch.Tensor, tar_pos: torch.Tensor) -> torch.Tensor:
    """compute_location_observations (humanoid_reach.py:224-236)."""
    return quat_rotate(heading_quat(root_states[:, 3:7], inverse=True), tar_pos - root_states[:, 0:3])


def reach_reward(reach_body_pos: torch.Tensor, tar_pos: torch.Tensor) -> torch.Tensor:
    """compute_reach_reward (humanoid_reach.py:238-250)."""
    d = tar_pos - reach_body_pos
    return torch.exp(-4.0 * torch.sum(d * d, dim=-1))


def pd_targets(action: torch.Tensor, offset: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """Humanoid._action_to_pd_targets (humanoid.py:1392-1394)."""
    return offset + scale * action


def humanoid_reset(progress_buf, contact_buf, contact_body_ids, rigid_body_pos, max_episode_length: int, enable_early_termination: bool,
                   termination_heights) -> Tuple[torch.Tensor, torch.Tensor]:
    """compute_humanoid_reset (humanoid.py:1573-1608): fall = contact force > 0.1 on a non-contact body AND a non-contact
    body below its termination height, only after progress > 1; reset also when the episode length is reached."""
    terminated = torch.zeros_like(progress_buf)
    if enable_early_termination:
        masked = contact_buf.clone()
        masked[:, contact_body_ids, :] = 0
        fall_contact = torch.any(torch.any(torch.abs(masked) > 0.1, dim=-1), dim=-1)
        fall_height = rigid_body_pos[..., 2] < termination_heights
        fall_height[:, contact_body_ids] = False
        has_fallen = fall_contact & torch.any(fall_height, dim=-1) & (progress_buf > 1)
        terminated = torch.where(has_fallen, torch.ones_like(progress_buf), terminated)
    reset = torch.where(progress_buf >= max_episode_length - 1, torch.ones_like(progress_buf), terminated)
    return reset, terminated


def speed_obs(root_states: torch.Tensor, tar_speed: torch.Tensor) -> torch.Tensor:
    """compute_speed_observations (humanoid_speed.py:310-325): heading-frame x axis (2) + target speed."""
    x = torch.zeros_like(root_states[:, 0:3])
    x[:, 0] = 1
    d = quat_rotate(heading_quat(root_states[:, 3:7], inverse=True), x)
    return torch.cat([d[:, 0:2], tar_speed[:, None]], dim=-1)


def speed_reward(root_pos, prev_root_pos, tar_speed, dt: float) -> torch.Tensor:
    """compute_speed_reward (humanoid_speed.py:327-343)."""
    v = (root_pos - prev_root_pos) / dt
    err = tar_speed - v[:, 0]
    return torch.exp(-0.25 * (err * err + 0.1 * v[:, 1] * v[:, 1]))


def power_reward(dof_force, dof_vel, progress_buf, coefficient: float) -> torch.Tensor:
    """humanoid_speed.py:215-222 (same expression as humanoid_im.py:910-917)."""
    p = -coefficient * torch.abs(dof_force * dof_vel).sum(dim=-1)
    p[progress_buf <= 3] = 0
    return p


def strike_obs(root_states: torch.Tensor, tar_states: torch.Tensor) -> torch.Tensor:
    """compute_strike_observations (humanoid_strike.py:270-293)."""
    hinv = heading_quat(root_states[:, 3:7], inverse=True)
    lp = tar_states[:, 0:3] - root_states[:, 0:3]
    lp[:, 2] = tar_states[:, 2]
    return torch.cat([quat_rotate(hinv, lp), quat_to_six(quat_mul(hinv, tar_states[:, 3:7])), quat_rotate(hinv, tar_states[:, 7:10]),
                      quat_rotate(hinv, tar_states[:, 10:13])], dim=-1)


def strike_reward(tar_pos, tar_rot, root_pos, prev_root_pos, dt: float) -> torch.Tensor:
    """compute_strike_reward (humanoid_strike.py:295-328)."""
    up = torch.zeros_like(tar_pos)
    up[:, 2] = 1
    rot_err = torch.sum(up * quat_rotate(tar_rot, up), dim=-1)
    rot_r = torch.clamp_min(1.0 - rot_err, 0.0)
    d = torch.nn.functional.normalize(tar_pos[:, 0:2] - root_pos[:, 0:2], dim=-1)
    v = (root_pos - prev_root_pos) / dt
    dir_speed = torch.sum(d * v[:, :2], dim=-1)
    verr = torch.clamp_min(1.0 - dir_speed, 0.0)
    vel_r = torch.exp(-4.0 * verr * verr)
    vel_r[dir_speed <= 0] = 0
    r = 0.6 * rot_r + 0.4 * vel_r
    return torch.where(rot_err < 0.2, torch.ones_like(r), r)


def strike_reset(progress_buf, contact_buf, contact_body_ids, rigid_body_pos, tar_contact_forces, strike_body_ids, max_episode_length: int,
                 enable_early_termination: bool, termination_heights) -> Tuple[torch.Tensor, torch.Tensor]:
    """The strike task's compute_humanoid_reset (humanoid_strike.py:330-375): fall as in humanoid_reset, OR the target pushed with more
    than 50 N (x / y) while a body that is neither a ground-contact nor a strike body carries more than 50 N."""
    terminated = torch.zeros_like(progress_buf)
    if enable_early_termination:
        masked = contact_buf.clone()
        masked[:, contact_body_ids, :] = 0
        fall_contact = torch.any(torch.any(torch.abs(masked) > 0.1, dim=-1), dim=-1)
        fall_height = rigid_body_pos[..., 2] < termination_heights
        fall_height[:, contact_body_ids] = False
        has_fallen = fall_contact & torch.any(fall_height, dim=-1)
        tar_contact = torch.any(torch.abs(tar_contact_forces[..., 0:2]) > 50.0, dim=-1)
        masked[:, strike_body_ids, :] = 0
        nonstrike = torch.any(torch.any(torch.abs(masked) > 50.0, dim=-1), dim=-1)
        failed = (has_fallen | (tar_contact & nonstrike)) & (progress_buf > 1)
        terminated = torch.where(failed, torch.ones_like(progress_buf), terminated)
    reset = torch.where(progress_buf >= max_episode_length - 1, torch.ones_like(progress_buf), terminated)
    return reset, terminated


# ------------------------------------------------------------------------------------------------
# MotionLib loader (SURVEY 8f-1): what `load_motions` computes per clip before concatenating the tables
# ------------------------------------------------------------------------------------------------
def _pl_quat_mul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """poselib rotation3d.quat_mul (:15-27), the 16-product Hamilton form (xyzw)."""
    x1, y1, z1, w1 = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    x2, y2, z2, w2 = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    w = w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2
    x = w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2
    y = w1 * y2 + y1 * w2 + z1 * x2 - x1 * z2
    z = w1 * z2 + z1 * w2 + x1 * y2 - y1 * x2
    return torch.stack([x, y, z, w], dim=-1)


def _pl_quat_normalize(q: torch.Tensor) -> torch.Tensor:
    """rotation3d.quat_normalize (:93-98): real part made non-negative (quat_pos, float mask), then unit length."""
    z = (q[..., 3:] < 0).float()
    q = (1 - 2 * z) * q
    return q / q.norm(p=2, dim=-1).unsqueeze(-1).clamp(min=1e-9)


def _pl_quat_mul_norm(a, b):
    return _pl_quat_normalize(_pl_quat_mul(a, b))


def _pl_quat_conj(q):
    return torch.cat([-q[..., :3], q[..., 3:]], dim=-1)


def _pl_quat_rotate(rot, vec):
    """rotation3d.quat_rotate (:206-211): imaginary part of rot (x) (vec, 0) (x) conj(rot)."""
    other = torch.cat([vec, torch.zeros_like(vec[..., :1])], dim=-1)
    return _pl_quat_mul(_pl_quat_mul(rot, other), _pl_quat_conj(rot))[..., :3]


def loader_heading(pose_aa, pose_quat_global, trans: torch.Tensor, heading: float):
    """Heading randomisation of motion_lib_smpl.py:131-140 for a given angle (the reference's own scipy calls)."""
    from scipy.spatial.transform import Rotation as sRot
    import numpy as np
    B, J, N = pose_quat_global.shape
    rot = sRot.from_euler("xyz", np.array([0.0, 0.0, heading]))
    pose_aa = torch.as_tensor(pose_aa).clone()
    pose_aa[:, :3] = torch.tensor((rot * sRot.from_rotvec(pose_aa[:, :3])).as_rotvec())
    pose_quat_global = (rot * sRot.from_quat(np.asarray(pose_quat_global).reshape(-1, 4))).as_quat().reshape(B, J, N)
    trans = torch.matmul(trans, torch.from_numpy(rot.as_matrix().T))
    return pose_aa, pose_quat_global, trans


def loader_clip(pose_quat_global, trans: torch.Tensor, fps: float, parents, local_translation) -> Dict[str, torch.Tensor]:
    """One clip through `SkeletonState.from_rotation_and_root_translation(is_local=False)` ->
    `SkeletonMotion.from_skeleton_state` -> `compute_motion_dof_vels` (motion_lib_smpl.py:147-150; poselib skeleton3d.py:389-462,
    :1000-1022, :1100-1118; motion_lib_base.py:47-70) in the reference's own mix of precisions: global rotations and angular
    velocities float64, local rotations / positions / linear and dof velocities float32; `load_motions` casts all to fp32 (:297-304).

    pose_quat_global [T, J, 4] xyzw (after the heading step), trans [T, 3] float64, parents [J], local_translation [J, 3]."""
    import numpy as np
    from scipy.ndimage import gaussian_filter1d
    g = torch.as_tensor(pose_quat_global, dtype=torch.float64)
    T, J = g.shape[0], g.shape[1]
    parents = [int(p) for p in parents]
    dt = 1 / fps
    # local rotations from the given global ones (skeleton3d.py:444-462): computed in float64 but ASSIGNED into a float32
    # identity tensor (quat_identity_like builds float32), so everything downstream of them is float32
    lr = torch.zeros(T, J, 4, dtype=torch.float32)
    lr[..., 3] = 1.0
    for j, p in enumerate(parents):
        lr[:, j] = (g[:, j] if p == -1 else _pl_quat_mul_norm(_pl_quat_conj(g[:, p]), g[:, j])).float()
    # forward kinematics for the joint positions (:389-407), float32: the skeleton's offsets and the root translation sit in
    # a float32 tensor (:478-481) next to the float32 local rotations
    loc = torch.as_tensor(local_translation).float()
    root = trans.float()
    rot_fk, pos = [None] * J, [None] * J
    for j, p in enumerate(parents):
        if p == -1:
            rot_fk[j], pos[j] = lr[:, j], root
        else:
            rot_fk[j] = _pl_quat_mul_norm(rot_fk[p], lr[:, j])
            pos[j] = _pl_quat_rotate(rot_fk[p], loc[j].expand(T, 3)) + pos[p]
    gts = torch.stack(pos, dim=1)
    # velocities: central differences + sigma = 2 gaussian along time (:1100-1107), float32 in / float32 out
    vel = np.gradient(gts.numpy(), axis=-3) / dt
    gvs = torch.from_numpy(gaussian_filter1d(vel, 2, axis=-3, mode="nearest")).to(gts)
    # angular velocities from consecutive global rotations (:1110-1118); the last frame gets the identity difference
    dq = torch.zeros_like(g)
    dq[..., 3] = 1.0
    dq[:-1] = _pl_quat_mul_norm(g[1:], _pl_quat_conj(g[:-1]))
    angle = (2 * dq[..., 3] ** 2 - 1).clamp(-1, 1).arccos()
    axis = dq[..., :3] / dq[..., :3].norm(p=2, dim=-1, keepdim=True).clamp(min=1e-9)
    gavs = torch.from_numpy(gaussian_filter1d((axis * angle.unsqueeze(-1) / dt).numpy(), 2, axis=-3, mode="nearest"))
    # dof velocities from consecutive LOCAL rotations, joints 1.. (motion_lib_base.py:47-70); the last frame repeats
    rows = []
    for f in range(T - 1):
        d_ang, d_axis = quat_to_angle_axis(quat_mul(quat_conj(lr[f]), lr[f + 1]))
        rows.append((d_axis * d_ang.unsqueeze(-1) / dt)[1:])
    rows.append(rows[-1])
    dvs = torch.stack(rows, dim=0)
    return {"gts": gts, "grs": g, "lrs": lr, "gvs": gvs, "gavs": gavs, "dvs": dvs}
