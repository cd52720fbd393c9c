"""Stand-in for the reference surface `HumanoidZTaskResetB200Mixin` builds on (TEST INFRASTRUCTURE): the tensors and methods of
Humanoid / HumanoidAMP / HumanoidReach / HumanoidSpeed / HumanoidStrike the reset touches, with Isaac-Gym shaped views (2 actors per
env, 72 dofs x (pos, vel), 26 bodies).  Isaac Gym is not installable, so the gym setters are recorded and the refresh copies back a
stale simulator copy of the rigid bodies before the `_reset_rb_*` restore, as `_refresh_sim_tensors` (humanoid_amp.py:598-620) does."""
import types

import torch

from oracle import pulse_oracle as po
from tests import ztask_reset_oracle as zo

OBS_SIZE = {"reach": 361, "speed": 361, "strike": 373}


class StandInZTask:
    def __init__(self, kind, motion_lib, device, n, state_init="Random", upright=True, seed=0):
        dev = torch.device(device)
        g = torch.Generator().manual_seed(seed)
        r = lambda *s: torch.randn(*s, generator=g).to(dev)
        self.device, self.num_envs, self.humanoid_type, self.amp_obs_v, self.dt = dev, n, "smpl", 1, zo.DT
        self._state_init = types.SimpleNamespace(name=state_init)
        self._motion_lib = motion_lib
        self.smpl_parser_n = self.smpl_parser_m = self.smpl_parser_f = zo.StandInParser()
        self.humanoid_shapes = torch.cat([torch.ones(n, 1), torch.linspace(-1.0, 1.0, 10).expand(n, 10)], dim=-1).to(dev)
        self._key_body_ids, self.dof_subset = torch.tensor(po.KEY_BODY_IDS, device=dev), po.amp_dof_subset().to(dev)
        self._has_dof_subset, self._has_upright_start, self._amp_root_height_obs, self._num_amp_obs_steps = True, upright, False, 10
        self._rigid_body_state_reshaped = r(n, 26, 13)
        rb = self._rigid_body_state_reshaped[:, :24]
        self._rigid_body_pos, self._rigid_body_rot, self._rigid_body_vel, self._rigid_body_ang_vel = rb[..., 0:3], rb[..., 3:7], rb[..., 7:10], rb[..., 10:13]
        self._dof_state = r(n, 72, 2)
        self._dof_pos, self._dof_vel = self._dof_state[:, :69, 0], self._dof_state[:, :69, 1]
        self._root_states = r(n, 2, 13)
        self._humanoid_root_states = self._root_states[:, 0]
        self._contact_forces = r(n, 26, 3)
        self._humanoid_actor_ids = (2 * torch.arange(n, device=dev)).to(torch.int32)
        self.progress_buf = torch.randint(0, 300, (n,), generator=g).to(dev)
        self.reset_buf, self._terminate_buf = torch.zeros(n, dtype=torch.int64, device=dev), torch.ones(n, dtype=torch.int64, device=dev)
        self._sampled_motion_ids, self._motion_start_times = torch.zeros(n, dtype=torch.int64, device=dev), torch.rand(n, generator=g).to(dev)
        self._amp_obs_buf = r(n, 10, 195)
        self.obs_buf = r(n, OBS_SIZE[kind])
        if kind == "reach":
            self._tar_pos, self._tar_change_steps = r(n, 3), torch.zeros(n, dtype=torch.int64, device=dev)
            self._tar_dist_max, self._tar_height_min, self._tar_height_max = zo.REACH["tar_dist_max"], zo.REACH["tar_height_min"], zo.REACH["tar_height_max"]
            self._tar_change_steps_min, self._tar_change_steps_max = zo.REACH["steps_min"], zo.REACH["steps_max"]
        elif kind == "speed":
            self._tar_speed, self._speed_change_steps, self.power_acc = r(n), torch.zeros(n, dtype=torch.int64, device=dev), r(n, 2)
            self._tar_speed_min, self._tar_speed_max = zo.SPEED["tar_speed_min"], zo.SPEED["tar_speed_max"]
            self._speed_change_steps_min, self._speed_change_steps_max = zo.SPEED["steps_min"], zo.SPEED["steps_max"]
        else:
            self._target_states, self._tar_actor_ids = self._root_states[:, 1], self._humanoid_actor_ids + 1
            self._near_prob, self._near_dist, self._tar_dist_min, self._tar_dist_max = (zo.STRIKE[k] for k in ("near_prob", "near_dist", "tar_dist_min", "tar_dist_max"))
        self._state_reset_happened = False
        self._reset_default_env_ids, self._reset_ref_env_ids = [], []
        self.gym_calls = []
        self._sim_rigid_body_state = self._rigid_body_state_reshaped.clone()        # what gym's refresh writes back

    def _reset_envs(self, env_ids):
        raise AssertionError("reference reset path reached")

    def _reset_env_tensors(self, env_ids):               # humanoid.py:589-609 (+ humanoid_strike.py:152-158), setters recorded
        self.gym_calls.append(("set_actor_root_state_tensor_indexed", self._humanoid_actor_ids[env_ids], len(env_ids)))
        self.gym_calls.append(("set_dof_state_tensor_indexed", self._humanoid_actor_ids[env_ids], len(env_ids)))
        self.progress_buf[env_ids] = 0
        self.reset_buf[env_ids] = 0
        self._terminate_buf[env_ids] = 0
        self._contact_forces[env_ids] = 0
        if hasattr(self, "_tar_actor_ids"):
            self.gym_calls.append(("set_actor_root_state_tensor_indexed", self._tar_actor_ids[env_ids], len(env_ids)))

    def _refresh_sim_tensors(self):                      # humanoid_amp.py:598-620
        self._rigid_body_state_reshaped.copy_(self._sim_rigid_body_state)
        if self._state_reset_happened and "_reset_rb_pos" in self.__dict__:
            env_ids = self._reset_ref_env_ids
            if len(env_ids) > 0:
                self._rigid_body_pos[env_ids] = self._reset_rb_pos
                self._rigid_body_rot[env_ids] = self._reset_rb_rot
                self._rigid_body_vel[env_ids] = self._reset_rb_vel
                self._rigid_body_ang_vel[env_ids] = self._reset_rb_ang_vel
                self._state_reset_happened = False
