"""CPU oracle of the latent-space tasks' reference-state reset (TEST INFRASTRUCTURE): `_sample_ref_state` of HumanoidReach /
HumanoidSpeed / HumanoidStrike with the SMPL ground fix (humanoid_amp.py:382-488, humanoid_reach.py:46-48, humanoid_speed.py:251-270,
humanoid_strike.py:147-150), `_set_env_state`, `_reset_target` (humanoid_strike.py:124-145), `_init_amp_obs` (humanoid_amp.py:519-563)
and `_reset_task` (humanoid_reach.py:134-146, humanoid_speed.py:166-175), restated over torch with the draws supplied by the caller.
Pinned to the unmodified reference by tests/golden/ztask_reset.npz (make_golden_ztask_reset.py).

The ground fix takes the per-frame floor table `pulse_b200.ztask_reset.smpl_ground_table` builds, as the kernel does.  SMPL model files
are not part of the project, so `StandInParser` supplies `get_joints_verts`: a seeded, pose-dependent point cloud whose root joint moves
with the body shape.  It pins how the table is derived, not real SMPL geometry."""
import math
from typing import Dict

import torch

from oracle import pulse_oracle as po
from oracle.terrain_oracle import quat_apply   # isaacgym.torch_utils.quat_apply

AS_IS, ROOT_XY_ZERO, FACE_X = 0, 1, 2
RANDOM, START = 0, 1
POSE_MODE = {"reach": ROOT_XY_ZERO, "strike": ROOT_XY_ZERO, "speed": FACE_X}
# task options of the fixture and the GPU tests (the reference defaults of env_pulse_amp.yaml / the task classes)
STRIKE = dict(near_prob=0.5, near_dist=1.5, tar_dist_min=0.5, tar_dist_max=10.0)
REACH = dict(tar_dist_max=1.0, tar_height_min=0.5, tar_height_max=1.5, steps_min=100, steps_max=200)
SPEED = dict(tar_speed_min=0.0, tar_speed_max=5.0, steps_min=100, steps_max=200)
DT = float(torch.tensor(1.0 / 60.0, dtype=torch.float32) * 2)
CLIPS, TABLE_SEED, PARSER_SEED = 7, 31, 32


class StandInParser:
    """`get_joints_verts(pose [B,72], th_betas [B,K], th_trans [B,3]) -> (vertices [B,64,3], joints [B,24,3])` of a seeded point cloud:
    rotated by the root's axis-angle, lifted by a pose-dependent term, joints offset by the shape; the translation moves both."""

    def __init__(self, seed: int = PARSER_SEED):
        g = torch.Generator().manual_seed(seed)
        self.points = torch.randn(64, 3, generator=g) * torch.tensor([0.25, 0.25, 0.7])
        self.lift = torch.randn(72, 64, generator=g) * 0.05
        self.joints = torch.randn(24, 3, generator=g) * 0.3
        self.shape = torch.randn(10, 3, generator=g) * 0.1

    @staticmethod
    def _rotation(aa):
        q = po.exp_map_to_quat(aa)
        eye = torch.eye(3).expand(aa.shape[0], 3, 3)
        return torch.stack([po.quat_rotate(q, eye[:, :, c]) for c in range(3)], dim=-1)

    def get_joints_verts(self, pose, th_betas, th_trans):
        dev = pose.device                                # computed on the CPU, returned where the caller's tensors live
        pose, th_betas, th_trans = pose.cpu(), th_betas.cpu(), th_trans.cpu()
        v, j = self._forward(pose, th_betas, th_trans)
        return v.to(dev), j.to(dev)

    def _forward(self, pose, th_betas, th_trans):
        R = self._rotation(pose[:, :3].float())
        v = torch.einsum("bij,vj->bvi", R, self.points)
        v = v + torch.stack([torch.zeros_like(v[..., 0]), torch.zeros_like(v[..., 0]), torch.tanh(pose.float() @ self.lift)], dim=-1)
        j = torch.einsum("bij,kj->bki", R, self.joints) + (th_betas[:, :10].float() @ self.shape)[:, None]
        return v + th_trans[:, None], j + th_trans[:, None]


def fixture_tables():
    """The motion tables and body shape of the fixture, rebuilt from seeds: `exact_tables(CLIPS)` and one gender-1 shape row."""
    from tests.helpers import exact_tables
    tb = exact_tables(CLIPS, seed=TABLE_SEED, min_frames=4, spread=40)
    betas = torch.linspace(-1.0, 1.0, 10)
    return tb, betas


def sample_ref_state(tb, motion_ids, phase, floor, pose_mode: int, upright: bool, state_init: int) -> Dict[str, torch.Tensor]:
    """`_sample_ref_state` for the clips `motion_ids` (one per reset env, compact) with the start-time uniforms `phase`."""
    n = motion_ids.shape[0]
    t0 = po.sample_time_interval(tb, motion_ids, phase) if state_init == RANDOM else torch.zeros(n)
    ms = po.motion_state(tb, motion_ids, t0)
    root_pos, rb_pos = ms["root_pos"].clone(), ms["rg_pos"].clone()
    f0 = ms["frame_idx0"] + tb.length_starts[motion_ids]
    d = (floor[f0] + root_pos[:, 2]) - 0.02                       # min_v (V - (J0 - root)).z - 0.02
    root_pos[:, 2] -= d
    rb_pos[..., 2] -= d[:, None]
    s = dict(motion_ids=motion_ids, t0=t0, root_pos=root_pos, root_rot=ms["root_rot"], root_vel=ms["root_vel"], root_ang_vel=ms["root_ang_vel"],
             dof_pos=ms["dof_pos"], dof_vel=ms["dof_vel"], rb_pos=rb_pos, rb_rot=ms["rb_rot"], body_vel=ms["body_vel"], body_ang_vel=ms["body_ang_vel"])
    if pose_mode == ROOT_XY_ZERO:
        s["root_pos"][:, :2] = 0.0
    elif pose_mode == FACE_X:
        h = po.heading_quat(s["root_rot"] if upright else po.remove_base_rot(s["root_rot"]), inverse=True)
        hr = h[:, None].expand(n, rb_pos.shape[1], 4)
        rp = s["root_pos"][:, None, :]
        s["root_rot"] = po.quat_mul(h, s["root_rot"])
        s["rb_pos"] = quat_apply(hr, s["rb_pos"] - rp) + rp
        s["rb_rot"] = po.quat_mul(hr, s["rb_rot"])
        s["root_ang_vel"] = quat_apply(h, s["root_ang_vel"])
        s["root_vel"] = quat_apply(h, s["root_vel"])
        s["body_vel"] = quat_apply(hr, s["body_vel"])
    return s


def reset_target(root_xy, u, near_prob, near_dist, tar_dist_min, tar_dist_max) -> torch.Tensor:
    """`_reset_target` with the uniforms u [n, 4] = (near, distance, bearing, yaw): the [n, 13] target root states."""
    n = u.shape[0]
    dist_max = tar_dist_max * torch.ones(n)
    dist_max[u[:, 0] < near_prob] = near_dist
    dist = (dist_max - tar_dist_min) * u[:, 1] + tar_dist_min
    theta, yaw = 2 * math.pi * u[:, 2], 2 * math.pi * u[:, 3]
    ts = torch.zeros(n, 13)
    ts[:, 0] = dist * torch.cos(theta) + root_xy[:, 0]
    ts[:, 1] = dist * torch.sin(theta) + root_xy[:, 1]
    ts[:, 2] = 0.9
    ts[:, 3:7] = po.quat_from_angle_axis(yaw, torch.tensor([0.0, 0.0, 1.0]).expand(n, 3))
    return ts


def amp_row(p, q, v, w, dof_pos, dof_vel, key_pos, upright: bool, width: int) -> torch.Tensor:
    """build_amp_observations_smpl with dof_subset; width 195 drops the root height."""
    q = q if upright else po.remove_base_rot(q)
    return po.amp_obs_smpl(p, q, v, w, dof_pos, dof_vel, key_pos, po.amp_dof_subset(), root_height_obs=width == po.AMP_OBS)


def amp_history(tb, s, body_state, dof_pos, dof_vel, steps: int, dt: float, upright: bool, width: int) -> torch.Tensor:
    """`_init_amp_obs`: row 0 from the written rigid bodies / dofs, rows k >= 1 from the unadjusted motion at t0 - k dt."""
    key = list(po.KEY_BODY_IDS)
    rows = [amp_row(body_state[:, 0, 0:3], body_state[:, 0, 3:7], body_state[:, 0, 7:10], body_state[:, 0, 10:13], dof_pos, dof_vel,
                    body_state[:, key, 0:3], upright, width)]
    for k in range(1, steps):
        h = po.motion_state(tb, s["motion_ids"], s["t0"] + (-dt) * k)
        rows.append(amp_row(h["root_pos"], h["root_rot"], h["root_vel"], h["root_ang_vel"], h["dof_pos"], h["dof_vel"], h["rg_pos"][:, key],
                            upright, width))
    return torch.stack(rows, dim=1)


def reach_task(u3, steps, progress, tar_dist_max, tar_height_min, tar_height_max, **_):
    rp = u3.clone()
    rp[:, 0:2] = tar_dist_max * (2.0 * rp[:, 0:2] - 1.0)
    rp[:, 2] = (tar_height_max - tar_height_min) * rp[:, 2] + tar_height_min
    return rp, progress + steps


def speed_task(u, steps, progress, tar_speed_min, tar_speed_max, **_):
    return (tar_speed_max - tar_speed_min) * u + tar_speed_min, progress + steps


def ztask_reset(tb, st: Dict[str, torch.Tensor], env_ids, draws: Dict[str, torch.Tensor], floor, kind: str, upright: bool = True,
                state_init: int = RANDOM, num_amp_steps: int = 10, width: int = 195, dt: float = DT) -> Dict[str, torch.Tensor]:
    """The device reset for the ascending `env_ids`, draws injected per ENV (motion_ids [N], phase [N], strike_u [N,4]).  st keys:
    root_states [N,13], dof_pos / dof_vel [N,69], body_state [N,24,13], sampled_motion_ids, motion_start_times, progress_buf, reset_buf,
    terminate_buf, contact_forces [N,B,3], amp_obs_buf [N,S,width], target_states [N,13] (strike).  Returns updated copies."""
    o = {k: v.clone() for k, v in st.items()}
    ids = env_ids.long()
    if ids.numel() == 0:
        return o
    s = sample_ref_state(tb, draws["motion_ids"][ids], draws["phase"][ids], floor, POSE_MODE[kind], upright, state_init)
    o["root_states"][ids] = torch.cat([s["root_pos"], s["root_rot"], s["root_vel"], s["root_ang_vel"]], dim=-1)
    o["dof_pos"][ids], o["dof_vel"][ids] = s["dof_pos"], s["dof_vel"]
    o["body_state"][ids] = torch.cat([s["rb_pos"], s["rb_rot"], s["body_vel"], s["body_ang_vel"]], dim=-1)
    o["sampled_motion_ids"][ids], o["motion_start_times"][ids] = s["motion_ids"], s["t0"]
    for k in ("progress_buf", "reset_buf", "terminate_buf", "contact_forces"):
        o[k][ids] = 0
    if kind == "strike":
        o["target_states"][ids] = reset_target(s["root_pos"][:, :2], draws["strike_u"][ids], **STRIKE)
    o["amp_obs_buf"][ids] = amp_history(tb, s, o["body_state"][ids], s["dof_pos"], s["dof_vel"], num_amp_steps, dt, upright, width)
    return o
