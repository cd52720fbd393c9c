"""CPU oracle of the pedestrian terrain task's reference-state reset (TEST INFRASTRUCTURE): HumanoidPedestrianTerrain's
`_reset_ref_state_init` (humanoid_pedestrian_terrain.py:527-589) with `_sample_ref_state` (:488-525), the spawn on the walkable table
(`Terrain.sample_valid_locations` :1175-1189, `get_center_heights` :690-716), `_set_env_state`, `_init_amp_obs` (humanoid_amp.py:519-563)
and `_reset_task` -> `TrajGenerator.reset` (traj_generator.py:57-112), restated over torch with the draws supplied by the caller.
Pinned to the unmodified reference by tests/golden/terrain_reset.npz (make_golden_terrain_reset.py).

The clip, start time, ground fix and AMP history are those of tests/ztask_reset_oracle.py (the terrain task's `_sample_ref_state`
always calls `_sample_time`, for StateInit Start too, and adjusts no pose); heights are oracle/terrain_oracle.py's."""
from typing import Dict

import numpy as np
import torch

from oracle import terrain_oracle as to
from tests import ztask_reset_oracle as zo

DT = zo.DT
HSCALE, VSCALE = 0.1, 0.005       # Terrain.__init__ (:1121-1122)
# env_pulse_terrain.yaml / humanoid_traj.py:110 trajectory options; episode length 300
TRAJ = dict(dtheta_max=2.0, speed_min=0.0, speed_max=3.0, accel_max=2.0, sharp_turn_prob=0.02)
TRAJ_DT = to.traj_params(300, DT)


def walkable_table(walkable_field: torch.Tensor, horizontal_scale: float, border: int):
    """Terrain.__init__ (:1160-1171): the cells with walkable_field == 0, scaled to metres, strictly inside `border` cells of the
    extreme walkable coordinates.  `border` = int(border_size / horizontal_scale).  Returns (coord_x_scale, coord_y_scale), fp32."""
    coord_x, coord_y = torch.where(walkable_field == 0)
    cx, cy = coord_x * horizontal_scale, coord_y * horizontal_scale
    b = border * horizontal_scale
    keep = torch.logical_and(torch.logical_and(cy < cy.max() - b, cx < cx.max() - b), torch.logical_and(cy > cy.min() + b, cx > cx.min() + b))
    return cx[keep], cy[keep]


def walkable_field(rows: int, cols: int, seed: int = 3) -> torch.Tensor:
    """A synthetic walkable mask for the fixture and the tests (0 = walkable): blocked strips and a random 30 %, from a numpy seed."""
    rng = np.random.default_rng(seed)
    w = (rng.random((rows, cols)) < 0.3).astype(np.int16)
    w[:, 100:110] = 1
    w[60:70, :] = 1
    return torch.from_numpy(w)


def spawn(hf, s: Dict[str, torch.Tensor], new_xy: torch.Tensor, center_pts, upright: bool, hscale=HSCALE, vscale=VSCALE) -> torch.Tensor:
    """:553-567 in place on the sampled state: root xy <- new_xy, root z += mean center height at the new root, rigid-body xy += the
    shift; the bodies' z stays (the lift goes to key_pos only).  Returns the center heights."""
    diff = new_xy - s["root_pos"][:, 0:2]
    s["root_pos"][:, 0:2] = new_xy
    ch = to.center_heights(hf, hscale, vscale, torch.cat([s["root_pos"], s["root_rot"]], dim=1), center_pts, upright).mean(dim=-1)
    s["root_pos"][:, 2] += ch
    s["rb_pos"][..., 0:2] += diff[:, None, :]
    return ch


def terrain_reset(tb, st: Dict[str, torch.Tensor], env_ids, draws: Dict[str, torch.Tensor], floor, hf, coord_x, coord_y, upright: bool = True,
                  num_amp_steps: int = 10, width: int = 196, dt: float = DT, center_pts=None) -> Dict[str, torch.Tensor]:
    """The device reset for the ascending `env_ids`, draws injected per ENV: motion_ids [N], phase [N], loc_ids [N] (walkable-table
    indices).  st keys: root_states [N,13], dof_pos / dof_vel [N,69], body_state [N,24,13], sampled_motion_ids, motion_start_times,
    progress_buf, reset_buf, terminate_buf, contact_forces [N,B,3], amp_obs_buf [N,S,width].  Returns updated copies, plus
    'center_height' [n] of the reset envs."""
    o = {k: v.clone() for k, v in st.items()}
    ids = env_ids.long()
    if ids.numel() == 0:
        return o
    center_pts = to.center_height_points() if center_pts is None else center_pts
    s = zo.sample_ref_state(tb, draws["motion_ids"][ids], draws["phase"][ids], floor, zo.AS_IS, upright, zo.RANDOM)
    loc = draws["loc_ids"][ids]
    o["center_height"] = spawn(hf, s, torch.stack([coord_x[loc], coord_y[loc]], dim=-1), center_pts, upright)
    o["root_states"][ids] = torch.cat([s["root_pos"], s["root_rot"], s["root_vel"], s["root_ang_vel"]], dim=-1)
    o["dof_pos"][ids], o["dof_vel"][ids] = s["dof_pos"], s["dof_vel"]
    o["body_state"][ids] = torch.cat([s["rb_pos"], s["rb_rot"], s["body_vel"], s["body_ang_vel"]], dim=-1)
    o["sampled_motion_ids"][ids], o["motion_start_times"][ids] = s["motion_ids"], s["t0"]
    for k in ("progress_buf", "reset_buf", "terminate_buf", "contact_forces"):
        o[k][ids] = 0
    o["amp_obs_buf"][ids] = zo.amp_history(tb, s, o["body_state"][ids], s["dof_pos"], s["dof_vel"], num_amp_steps, dt, upright, width)
    return o


def reset_task(verts: torch.Tensor, env_ids, root_states: torch.Tensor, rand: torch.Tensor) -> torch.Tensor:
    """`_reset_task` (:480-485) of the reset envs from their new roots, draws per ENV [N, TRAJ_DRAWS]; returns updated waypoints."""
    v = verts.clone()
    ids = env_ids.long()
    if ids.numel():
        to.traj_reset(v, ids, root_states[ids, 0:3], rand[ids], TRAJ_DT, **TRAJ)
    return v
