"""Downstream latent-space reach task (SURVEY K21, BASELINE config 5): host-side mirror of
`phc.env.tasks.humanoid_reach.HumanoidReach` / `HumanoidReachZ` (humanoid_reach.py:17-166, :224-250) for the
post-physics path -- reward, reset, observation -- and the target resampling of `_update_task` / `_reset_task`.

The policy acts in the frozen PULSE latent space: `HumanoidReachZ.step -> step_z` decodes the 32-d action through the
prior + decoder (`pulse_b200.vae.PulseVAE.compute_z_actions`) before `pre_physics_step` maps it to PD targets
(`pulse_b200.vae.pd_targets`).  Isaac Gym keeps the physics and owns the state tensors, which are read in place.
"""
import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib

REACH_OBS = 361   # 358 self observation + 3 (target offset in the heading frame), humanoid_reach.py:69-74
# SMPL humanoid body order (smpl_humanoid.xml); contact bodies of the reach configs = both ankles and toes
SMPL_BODY_NAMES = ['Pelvis', 'L_Hip', 'L_Knee', 'L_Ankle', 'L_Toe', 'R_Hip', 'R_Knee', 'R_Ankle', 'R_Toe', 'Torso', 'Spine', 'Chest', 'Neck',
                   'Head', 'L_Thorax', 'L_Shoulder', 'L_Elbow', 'L_Wrist', 'L_Hand', 'R_Thorax', 'R_Shoulder', 'R_Elbow', 'R_Wrist', 'R_Hand']


class ReachTaskB200:
    kind, obs_size = _lib.ZTASK_REACH, REACH_OBS

    def __init__(self, num_envs: int, device="cuda:0", reach_body_name: str = "R_Hand", contact_bodies: Sequence[str] = ("R_Ankle", "L_Ankle", "R_Toe", "L_Toe"),
                 tar_change_steps_min: int = 100, tar_change_steps_max: int = 200, tar_dist_max: float = 1.0, tar_height_min: float = 0.5,
                 tar_height_max: float = 1.5, max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15):
        self.device = torch.device(device)
        self.num_envs = num_envs
        self.reach_body_id = SMPL_BODY_NAMES.index(reach_body_name)
        self.contact_body_mask = 0
        for n in contact_bodies:
            self.contact_body_mask |= 1 << SMPL_BODY_NAMES.index(n)
        self.tar_change_steps_min, self.tar_change_steps_max = tar_change_steps_min, tar_change_steps_max
        self.tar_dist_max, self.tar_height_min, self.tar_height_max = tar_dist_max, tar_height_min, tar_height_max
        self.max_episode_length, self.enable_early_termination = max_episode_length, enable_early_termination
        dev = self.device
        self.termination_heights = torch.full((24,), termination_height, device=dev)
        self._tar_pos = torch.zeros(num_envs, 3, device=dev)
        self._tar_change_steps = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self.obs_buf = torch.zeros(num_envs, REACH_OBS, device=dev)
        self.rew_buf = torch.zeros(num_envs, device=dev)
        self.reset_buf = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self._terminate_buf = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self._rand = torch.zeros(num_envs, 3, device=dev)
        self._steps = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self.lib = _lib.load()

    def get_task_obs_size(self) -> int:
        return 3

    def update_task(self, progress_buf: torch.Tensor, rand01: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None) -> None:
        """_update_task (:126-131): resample the target of every env whose progress reached `_tar_change_steps`.
        The uniform draws can be injected (tests); by default they are drawn for all envs on the device (the reference draws
        only for the selected subset -- same distribution, different random stream)."""
        if rand01 is None:
            rand01 = self._rand.uniform_()
        if steps is None:
            steps = self._steps.random_(self.tar_change_steps_min, self.tar_change_steps_max)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_reach_update_task(progress_buf.data_ptr(), self._tar_change_steps.data_ptr(), self._tar_pos.data_ptr(),
                                                        rand01.data_ptr(), steps.data_ptr(), self.tar_dist_max, self.tar_height_min, self.tar_height_max,
                                                        self.num_envs, _lib.current_stream(self.device)), "pulse_reach_update_task")

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_reward + _compute_reset + _compute_observations (humanoid.py:1315-1330 order) in one launch.
        rigid_body_state fp32 [N, B_env >= 24, 13] (Isaac Gym view, read in place); contact_forces fp32 [N, B_env, 3]."""
        a = self._step_args(rigid_body_state, progress_buf, contact_forces)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_reach_step(C.byref(a), self.num_envs, _lib.current_stream(self.device)), "pulse_reach_step")

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count) (int64 list, int32 device-side count): the rows
        post_physics_step writes for them, bit for bit, and nothing else."""
        a = self._step_args(rigid_body_state, progress_buf, contact_forces)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_reach_obs_list(C.byref(a), env_list.data_ptr(), count.data_ptr(), self.num_envs,
                                                     _lib.current_stream(self.device)), "pulse_reach_obs_list")

    def _step_args(self, rigid_body_state, progress_buf, contact_forces):
        return _lib.ReachStepArgs(
            body_state=rigid_body_state.data_ptr(), body_env_stride=rigid_body_state.stride(0),
            contact_forces=contact_forces.data_ptr() if contact_forces is not None else None,
            contact_env_stride=contact_forces.stride(0) if contact_forces is not None else 0,
            termination_heights=self.termination_heights.data_ptr(), tar_pos=self._tar_pos.data_ptr(), progress_buf=progress_buf.data_ptr(),
            contact_body_mask=self.contact_body_mask, reach_body_id=self.reach_body_id, enable_early_termination=int(self.enable_early_termination),
            max_episode_length=self.max_episode_length, obs_buf=self.obs_buf.data_ptr(), obs_stride=self.obs_buf.stride(0),
            rew_buf=self.rew_buf.data_ptr(), reset_buf=self.reset_buf.data_ptr(), terminate_buf=self._terminate_buf.data_ptr())
