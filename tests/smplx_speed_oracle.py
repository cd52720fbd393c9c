"""Restatements of the PULSE-X speed task (52-body SMPL-X humanoid, has_upright_start False) on top of oracle/pulse_oracle.py, and the
seeded synthetic 52-body MotionLib tables the device tests load."""
import torch

from oracle import pulse_oracle as po

BODIES, DOFS, SELF_OBS, SPEED_OBS = 52, 153, 778, 781


def self_obs(body_state: torch.Tensor, upright: bool = False) -> torch.Tensor:
    """compute_humanoid_observations_smpl_max (humanoid.py:1675-1731), local root obs and root height, no shape obs: the heading of
    remove_base_rot(root) unless `upright`.  [h | R(p_j - p_0) j >= 1 | six(hinv q_j) | R v_j | R w_j]."""
    pos, rot, vel, ang = body_state[..., 0:3], body_state[..., 3:7], body_state[..., 7:10], body_state[..., 10:13]
    n, nb, _ = pos.shape
    root_rot = rot[:, 0] if upright else po.remove_base_rot(rot[:, 0])
    hinv = po.heading_quat(root_rot, inverse=True).unsqueeze(1).expand(n, nb, 4)
    rel = po.quat_rotate(hinv, pos - pos[:, :1]).reshape(n, -1)[:, 3:]
    rot6 = po.quat_to_six(po.quat_mul(hinv, rot)).reshape(n, -1)
    return torch.cat([pos[:, 0, 2:3], rel, rot6, po.quat_rotate(hinv, vel).reshape(n, -1), po.quat_rotate(hinv, ang).reshape(n, -1)], dim=-1)


def speed_reward(root_pos, prev_root_pos, tar_speed, dt: float) -> torch.Tensor:
    """compute_speed_reward (humanoid_speed.py:327-343) in the kernel's fp32 operation order."""
    v = (root_pos - prev_root_pos) / torch.tensor(dt, dtype=torch.float32)
    err = tar_speed - v[:, 0]
    return torch.exp(-0.25 * (err * err + 0.1 * v[:, 1] * v[:, 1]))


def step(z: dict, contact_ids, max_len: int, dt: float):
    """The SMPL-X speed step of the inputs `z` (make_golden_smplx_speed.inputs' keys): (obs [N, 781], reward, reset, terminate)."""
    bs, root = z["body_state"], z["body_state"][:, 0]
    obs = torch.cat([self_obs(bs), po.speed_obs(root, z["tar_speed"])], dim=-1)
    rew = speed_reward(root[:, 0:3], z["prev_root_pos"], z["tar_speed"], dt)
    rs, tm = po.humanoid_reset(z["progress_buf"], z["contact_forces"], torch.as_tensor(contact_ids), bs[..., 0:3], max_len, True,
                               z["termination_heights"])
    return obs, rew, rs, tm


def tables(clips: int, seed: int, min_frames: int = 4, spread: int = 60) -> po.MotionTables:
    """Seeded 52-body MotionLib tables: unit global / local rotations, 30 fps clips of min_frames .. min_frames + spread frames."""
    g = torch.Generator().manual_seed(seed)
    nf = torch.randint(min_frames, min_frames + spread, (clips,), generator=g)
    F = int(nf.sum())
    unit = lambda q: q / q.norm(dim=-1, keepdim=True)
    dt = torch.full((clips,), 1.0 / 30.0)
    return po.MotionTables(
        gts=torch.randn(F, BODIES, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9]), grs=unit(torch.randn(F, BODIES, 4, generator=g)),
        lrs=unit(torch.randn(F, BODIES, 4, generator=g)), gvs=torch.randn(F, BODIES, 3, generator=g), gavs=torch.randn(F, BODIES, 3, generator=g),
        dvs=torch.randn(F, BODIES - 1, 3, generator=g), motion_aa=0.3 * torch.randn(F, 3 * BODIES, generator=g), lengths=dt * (nf - 1).float(), num_frames=nf,
        dt=dt, length_starts=torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(nf, 0)[:-1]]))


def ground_table(tb: po.MotionTables, parser, betas: torch.Tensor) -> torch.Tensor:
    """The per-frame floor table of `tb` for the seeded stand-in SMPL parser (tests/ztask_reset_oracle.py), which reads the first 72
    pose columns: min_v V_z - J0_z of each frame's pose at zero translation."""
    F = tb.motion_aa.shape[0]
    v, j = parser.get_joints_verts(tb.motion_aa[:, :72], betas.reshape(1, -1).expand(F, -1), torch.zeros(F, 3))
    return v[..., 2].min(dim=-1).values - j[:, 0, 2]


class Parser72:
    """The stand-in SMPL parser fed the first 72 columns of a 156-wide SMPL-X pose (its pose-dependent lift is 72 wide)."""

    def __init__(self, parser):
        self.parser = parser

    def get_joints_verts(self, pose, th_betas, th_trans):
        return self.parser.get_joints_verts(pose[:, :72], th_betas, th_trans)


def table_dict(tb: po.MotionTables) -> dict:
    return {k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "lengths", "num_frames", "dt", "length_starts")}
