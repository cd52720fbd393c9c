"""CPU oracle for the pedestrian terrain task HumanoidPedestrianTerrain(Z) (TEST INFRASTRUCTURE -- never imported by pulse_b200/).

fp32 PyTorch-CPU restatement of phc/env/tasks/humanoid_pedestrian_terrain.py and the trajectory generator
(phc/env/util/traj_generator.py, the copy humanoid_traj.py imports; same arithmetic as phc/utils/traj_generator.py), written
from the cited functions with their operation order, so that it reproduces the integer outputs (height-map cells, reset masks,
trajectory segments) of the reference.  Pinned against tests/golden/terrain.npz by tests/test_terrain_cpu.py.

Third-party arithmetic restated [3P-memory]: isaacgym.torch_utils.quat_apply.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from oracle.pulse_oracle import heading_quat, quat_mul, quat_rotate, quat_to_six, remove_base_rot, self_obs_smpl_max

TRAJ_VERTS = 101
TRAJ_DRAWS = 4 * (TRAJ_VERTS - 1) + 2


def center_height_points() -> torch.Tensor:
    """init_center_height_points (:591-606): the 3 x 3 grid x in +-0.1, y in +-0.2, [9, 3]."""
    gx, gy = torch.meshgrid(torch.tensor(np.linspace(-0.1, 0.1, 3)), torch.tensor(np.linspace(-0.2, 0.2, 3)), indexing="ij")
    p = torch.zeros(9, 3)
    p[:, 0], p[:, 1] = gx.flatten(), gy.flatten()
    return p


def square_height_points(extent: float = 2.0, res: int = 32) -> torch.Tensor:
    """init_square_height_points (:608-626): res x res grid over +-extent, [res * res, 3]."""
    v = torch.tensor(np.linspace(-extent, extent, res))
    gx, gy = torch.meshgrid(v, v, indexing="ij")
    p = torch.zeros(res * res, 3)
    p[:, 0], p[:, 1] = gx.flatten(), gy.flatten()
    return p


def quat_apply(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """isaacgym.torch_utils.quat_apply [3P-memory]."""
    shape = b.shape
    a, b = a.reshape(-1, 4), b.reshape(-1, 3)
    xyz = a[:, :3]
    t = xyz.cross(b, dim=-1) * 2
    return (b + a[:, 3:] * t + xyz.cross(t, dim=-1)).view(shape)


def quat_apply_yaw(quat: torch.Tensor, vec: torch.Tensor) -> torch.Tensor:
    """quat_apply_yaw (:1571-1576)."""
    q = quat.clone().view(-1, 4)
    q[:, :2] = 0.0
    q = q / q.norm(p=2, dim=-1).clamp(min=1e-9).unsqueeze(-1)
    return quat_apply(q, vec)


def world_points_to_map(points: torch.Tensor, hscale: float, rows: int, cols: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Terrain.world_points_to_map (:1191-1197): truncating fp32 division, clip to [0, dim - 2]."""
    p = (points / hscale).long()
    return torch.clip(p[..., 0].reshape(-1), 0, rows - 2), torch.clip(p[..., 1].reshape(-1), 0, cols - 2)


def sample_height_points(hf: Optional[torch.Tensor], points: torch.Tensor, hscale: float, vscale: float) -> torch.Tensor:
    """Terrain.sample_height_points (:1200-1267) without group / velocity maps; a plane (hf None) is flat 0.  [B, N]."""
    if hf is None:
        return torch.zeros(points.shape[:-1])
    px, py = world_points_to_map(points, hscale, hf.shape[0], hf.shape[1])
    return (torch.min(hf[px, py], hf[px + 1, py + 1]) * vscale).view(points.shape[:-1])


def center_points_world(root_states: torch.Tensor, pts: torch.Tensor, upright: bool) -> torch.Tensor:
    q = root_states[:, 3:7] if upright else remove_base_rot(root_states[:, 3:7])
    n = root_states.shape[0]
    return quat_apply_yaw(q.repeat(1, pts.shape[0]), pts.expand(n, -1, -1).contiguous()) + root_states[:, :3].unsqueeze(1)


def grid_points_world(root_states: torch.Tensor, pts: torch.Tensor, upright: bool) -> torch.Tensor:
    q = root_states[:, 3:7] if upright else remove_base_rot(root_states[:, 3:7])
    h = heading_quat(q)
    n = root_states.shape[0]
    return quat_apply(h.repeat(1, pts.shape[0]).reshape(-1, 4), pts.expand(n, -1, -1).contiguous()) + root_states[:, :3].unsqueeze(1)


def center_heights(hf, hscale, vscale, root_states, pts, upright: bool) -> torch.Tensor:
    """get_center_heights (:690-716)."""
    return sample_height_points(hf, center_points_world(root_states, pts, upright), hscale, vscale)


def grid_heights(hf, hscale, vscale, root_states, pts, upright: bool) -> torch.Tensor:
    """get_heights (:718-772) without the velocity map / group points."""
    return sample_height_points(hf, grid_points_world(root_states, pts, upright), hscale, vscale)


def traj_calc_pos(verts: torch.Tensor, traj_ids: torch.Tensor, times: torch.Tensor, traj_dt: float) -> torch.Tensor:
    """TrajGenerator.calc_pos (traj_generator.py:148-165); the phase divides by num_verts * dt, as in the reference."""
    nv = verts.shape[1]
    phase = torch.clip(times / (nv * traj_dt), 0.0, 1.0)
    seg = phase * (nv - 1)
    i0, i1 = torch.floor(seg).long(), torch.ceil(seg).long()
    lerp = (seg - i0).unsqueeze(-1)
    flat = verts.reshape(-1, 3)
    return (1.0 - lerp) * flat[traj_ids * nv + i0] + lerp * flat[traj_ids * nv + i1]


def traj_reset(verts: torch.Tensor, env_ids: torch.Tensor, init_pos: torch.Tensor, draws: torch.Tensor, traj_dt: float,
               dtheta_max: float, speed_min: float, speed_max: float, accel_max: float, sharp_turn_prob: float) -> None:
    """TrajGenerator.reset (traj_generator.py:57-112) with the uniform draws injected in the layout of pulse_traj_reset
    ([turn | sharp angle | sharp coin | speed change] x S, heading, initial speed); the bernoulli draw is u < sharp_turn_prob."""
    s = verts.shape[1] - 1
    dtheta = 2 * draws[:, 0:s] - 1.0
    dtheta *= dtheta_max * traj_dt
    dtheta_sharp = np.pi * (2 * draws[:, s:2 * s] - 1.0)
    sharp = draws[:, 2 * s:3 * s] < sharp_turn_prob
    dtheta[sharp] = dtheta_sharp[sharp]
    dtheta[:, 0] = np.pi * (2 * draws[:, 4 * s] - 1.0)
    dspeed = 2 * draws[:, 3 * s:4 * s] - 1.0
    dspeed *= accel_max * traj_dt
    dspeed[:, 0] = (speed_max - speed_min) * draws[:, 4 * s + 1] + speed_min
    speed = torch.zeros_like(dspeed)
    speed[:, 0] = dspeed[:, 0]
    for i in range(1, s):
        speed[:, i] = torch.clip(speed[:, i - 1] + dspeed[:, i], speed_min, speed_max)
    dtheta = torch.cumsum(dtheta, dim=-1)
    seg_len = speed * traj_dt
    dpos = torch.stack([torch.cos(dtheta), -torch.sin(dtheta), torch.zeros_like(dtheta)], dim=-1)
    dpos *= seg_len.unsqueeze(-1)
    dpos[..., 0, 0:2] += init_pos[..., 0:2]
    verts[env_ids, 0, 0:2] = init_pos[..., 0:2]
    verts[env_ids, 1:] = torch.cumsum(dpos, dim=-2)


def terrain_reward(root_pos, tar_pos, dof_force, dof_vel, fuzzy: bool, power_reward: bool, power_coefficient: float):
    """_compute_reward (:871-896) -> (rew, reward_raw [N, 2])."""
    d = tar_pos[..., 0:2] - root_pos[..., 0:2]
    err = torch.sum(d * d, dim=-1)
    if fuzzy:
        err[err < 0.0025] = 0
    loc = torch.exp(-2.0 * err)
    power = -power_coefficient * torch.abs(torch.multiply(dof_force, dof_vel)).sum(dim=-1)
    rew = loc + power if power_reward else loc
    return rew, torch.cat([loc[:, None], power[:, None]], dim=-1)


def terrain_reset(progress_buf, contact_buf, contact_body_ids, rigid_body_pos, tar_pos, max_episode_length: int, fail_dist: float,
                  enable_early_termination: bool, no_collision_check: bool):
    """compute_humanoid_reset (:1477-1531) -> (reset, terminated)."""
    terminated = torch.zeros_like(progress_buf)
    if enable_early_termination:
        masked = contact_buf.clone()
        masked[:, contact_body_ids, :] = 0
        fallen = (torch.sqrt(torch.square(torch.abs(masked.sum(dim=-2))).sum(dim=-1)) > 50) & (progress_buf > 1)
        delta = tar_pos[..., 0:2] - rigid_body_pos[..., 0, 0:2]
        far = torch.sum(delta * delta, dim=-1) > fail_dist * fail_dist
        failed = fallen | far
        if no_collision_check:
            failed[:] = False
        terminated = torch.where(failed, torch.ones_like(progress_buf), terminated)
    reset = torch.where(progress_buf >= max_episode_length - 1, torch.ones_like(progress_buf), terminated)
    return reset, terminated


def terrain_self_obs(hf, hscale, vscale, body_state, center_pts, upright: bool) -> torch.Tensor:
    """_compute_humanoid_obs (:195-223): z minus the mean center height around the rigid-body root, then the self observation."""
    pos = body_state[..., 0:3].clone()
    c = center_heights(hf, hscale, vscale, torch.cat([pos[:, 0], body_state[:, 0, 3:7]], dim=-1), center_pts, upright).mean(dim=-1, keepdim=True)
    pos[:, :, 2] = pos[:, :, 2] - c
    rot = body_state[..., 3:7]
    if upright:
        return self_obs_smpl_max(pos, rot, body_state[..., 7:10], body_state[..., 10:13])
    # heading of remove_base_rot(root) (humanoid.py:1681-1683); the body rotations are not rebased
    n, nb, _ = pos.shape
    hinv = heading_quat(remove_base_rot(rot[:, 0]), inverse=True).unsqueeze(1).expand(n, nb, 4)
    rel = quat_rotate(hinv, pos - pos[:, :1]).reshape(n, -1)[:, 3:]
    return torch.cat([pos[:, 0, 2:3], rel, quat_to_six(quat_mul(hinv, rot)).reshape(n, -1),
                      quat_rotate(hinv, body_state[..., 7:10]).reshape(n, -1), quat_rotate(hinv, body_state[..., 10:13]).reshape(n, -1)], dim=-1)


def terrain_task_obs(hf, hscale, vscale, root_states, head_pose, traj_samples, height_pts, center_pts, upright: bool,
                     use_center_height: bool = True) -> torch.Tensor:
    """_compute_task_obs (:385-440): compute_location_observations (:1588-1616) + the head-pose height map."""
    rot = root_states[:, 3:7] if upright else remove_base_rot(root_states[:, 3:7])
    hinv = heading_quat(rot, inverse=True).unsqueeze(1).expand(-1, traj_samples.shape[1], 4)
    loc = quat_rotate(hinv, traj_samples - root_states[:, None, 0:3])[..., 0:2].reshape(root_states.shape[0], -1)
    measured = grid_heights(hf, hscale, vscale, head_pose, height_pts, upright)
    if use_center_height:
        ref = center_heights(hf, hscale, vscale, root_states, center_pts, upright).mean(dim=-1, keepdim=True)
    else:
        ref = root_states[:, 2:3]
    return torch.cat([loc, torch.clip(ref - measured, -3, 3.0) * 5], dim=1)


def traj_sample_times(progress_buf, dt: float, num_samples: int = 10, sample_timestep: float = 0.5) -> torch.Tensor:
    """HumanoidTraj._fetch_traj_samples (humanoid_traj.py:196-211): progress * dt + k * trajSampleTimestep, [N, T]."""
    return (progress_buf * dt).unsqueeze(-1) + torch.arange(num_samples, dtype=torch.float) * sample_timestep


def fetch_traj_samples(verts, progress_buf, dt: float, traj_dt: float, num_samples: int = 10, sample_timestep: float = 0.5):
    t = traj_sample_times(progress_buf, dt, num_samples, sample_timestep)
    ids = torch.arange(verts.shape[0]).unsqueeze(-1).expand_as(t)
    return traj_calc_pos(verts, ids.flatten(), t.flatten(), traj_dt).view(verts.shape[0], num_samples, 3)


HEAD_BODY_ID = 13   # "Head" in the SMPL body order


def terrain_step(hf, hscale, vscale, body_state, root_states, progress_buf, contact_forces, contact_body_ids, dof_force, dof_vel, verts,
                 *, dt: float, traj_dt: float, max_episode_length: int, upright: bool = True, fuzzy: bool = False, power_reward: bool = False,
                 power_coefficient: float = 0.0005, fail_dist: float = 4.0, enable_early_termination: bool = True,
                 no_collision_check: bool = False, use_center_height: bool = True, height_pts=None, center_pts=None):
    """post_physics_step of the task in the reference's order: reward, reset, observation.  Returns a dict."""
    height_pts = square_height_points() if height_pts is None else height_pts
    center_pts = center_height_points() if center_pts is None else center_pts
    n = body_state.shape[0]
    tar = traj_calc_pos(verts, torch.arange(n), progress_buf * dt, traj_dt)
    rew, raw = terrain_reward(root_states[:, 0:3], tar, dof_force, dof_vel, fuzzy, power_reward, power_coefficient)
    reset, term = terrain_reset(progress_buf, contact_forces, contact_body_ids, body_state[..., 0:3], tar, max_episode_length, fail_dist,
                                enable_early_termination, no_collision_check)
    self_obs = terrain_self_obs(hf, hscale, vscale, body_state, center_pts, upright)
    head = body_state[:, HEAD_BODY_ID, 0:7]
    task_obs = terrain_task_obs(hf, hscale, vscale, root_states, head, fetch_traj_samples(verts, progress_buf, dt, traj_dt), height_pts,
                                center_pts, upright, use_center_height)
    return dict(rew=rew, reward_raw=raw, reset=reset, terminate=term, obs=torch.cat([self_obs, task_obs], dim=-1))


def traj_params(max_episode_length: int, dt: float, num_verts: int = TRAJ_VERTS) -> float:
    """HumanoidTraj._build_traj_generator (humanoid_traj.py:106-114) + TrajGenerator.__init__: dt = episode_dur / (num_verts - 1)."""
    return max_episode_length * dt / (num_verts - 1)
