"""fp32 restatements of the PULSE-X reach and strike steps (52-body SMPL-X humanoid, has_upright_start False) on top of
oracle/pulse_oracle.py and tests/smplx_speed_oracle.py, pinned to the reference by tests/golden/smplx_target.npz."""
import torch

from oracle import pulse_oracle as po
from tests import smplx_speed_oracle as so

REACH_OBS, STRIKE_OBS = 781, 793


def step(z: dict, kind: str, contact_ids, max_len: int, dt: float, reach_id: int = 36, strike_ids=(35, 36, 45)):
    """The SMPL-X reach / strike step of the inputs `z` (make_golden_smplx_target.inputs' keys): (obs [N, 781 | 793], reward, reset,
    terminate).  The self observation takes the heading of remove_base_rot(root), the task observation that of the raw root."""
    bs, root = z["body_state"], z["body_state"][:, 0]
    pos = bs[..., 0:3]
    if kind == "reach":
        obs = torch.cat([so.self_obs(bs), po.reach_obs(root, z["tar_pos"])], dim=-1)
        rew = po.reach_reward(pos[:, reach_id], z["tar_pos"])
        rs, tm = po.humanoid_reset(z["progress_buf"], z["contact_forces"], torch.as_tensor(contact_ids), pos, max_len, True, z["termination_heights"])
    else:
        ts = z["target_states"]
        obs = torch.cat([so.self_obs(bs), po.strike_obs(root, ts)], dim=-1)
        rew = po.strike_reward(ts[:, 0:3], ts[:, 3:7], root[:, 0:3], z["prev_root_pos"], dt)
        rs, tm = po.strike_reset(z["progress_buf"], z["contact_forces"], torch.as_tensor(contact_ids), pos, z["tar_contact_forces"],
                                 torch.as_tensor(strike_ids), max_len, True, z["termination_heights"])
    return obs, rew, rs, tm
