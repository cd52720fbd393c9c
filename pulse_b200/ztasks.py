"""Downstream latent-space speed and strike tasks (SURVEY 8f-4): host-side mirrors of `HumanoidSpeed(Z)` / `HumanoidStrike(Z)`
(phc/env/tasks/humanoid_speed.py, humanoid_strike.py) for the post-physics path -- reward, reset, observation in ONE launch
(`pulse_ztask_step`) -- and the task-state updates (`_update_task` / `_reset_task`).  Like the reach task (pulse_b200/reach.py) the policy
acts in the frozen PULSE latent space (`PulseVAE.compute_z_actions`); Isaac Gym keeps the physics and owns the state tensors.
`SmplxSpeedTaskB200` is the speed task of PULSE-X on the 52-body SMPL-X humanoid (`pulse_smplx_speed_step`); `SmplxReachTaskB200` and
`SmplxStrikeTaskB200` are its reach and strike tasks (`pulse_smplx_target_step`).
"""
import ctypes as C
import math
from typing import Optional, Sequence

import torch

from . import _lib
from .reach import SMPL_BODY_NAMES, ReachTaskB200

SPEED_OBS, STRIKE_OBS = 361, 373      # 358 self observation + 3 / + 15


def _mask(names: Sequence[str]) -> int:
    m = 0
    for n in names:
        m |= 1 << SMPL_BODY_NAMES.index(n)
    return m


class _ZTaskBase:
    kind, obs_size = 0, 0

    def __init__(self, num_envs: int, device, contact_bodies, max_episode_length: int, enable_early_termination: bool, termination_height: float,
                 dt: float):
        self.device, self.num_envs = torch.device(device), int(num_envs)
        self.contact_body_mask = _mask(contact_bodies)
        self.strike_body_mask = 0
        self.max_episode_length, self.enable_early_termination, self.dt = int(max_episode_length), bool(enable_early_termination), float(dt)
        dev = self.device
        self.termination_heights = torch.full((24,), termination_height, device=dev)
        self._prev_root_pos = torch.zeros(num_envs, 3, device=dev)
        self.obs_buf = torch.zeros(num_envs, self.obs_size, device=dev)
        self.rew_buf = torch.zeros(num_envs, device=dev)
        self.reset_buf = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self._terminate_buf = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self.lib = _lib.load()

    def pre_physics_step(self, root_states: torch.Tensor) -> None:
        """`self._prev_root_pos[:] = self._humanoid_root_states[..., 0:3]` (humanoid_speed.py:73-76, humanoid_strike.py pre_physics_step)."""
        self._prev_root_pos.copy_(root_states[:, 0:3])

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        if rigid_body_state.dim() != 3 or rigid_body_state.shape[1] < 24 or rigid_body_state.stride(1) != 13 or rigid_body_state.stride(2) != 1:
            raise _lib.PulseError("rigid_body_state must be a [N, B>=24, 13] view with row stride 13")
        return _lib.ZTaskStepArgs(
            kind=self.kind, enable_early_termination=int(self.enable_early_termination), body_state=rigid_body_state.data_ptr(),
            body_env_stride=rigid_body_state.stride(0), contact_forces=contact_forces.data_ptr() if contact_forces is not None else None,
            contact_env_stride=contact_forces.stride(0) if contact_forces is not None else 0, termination_heights=self.termination_heights.data_ptr(),
            contact_body_mask=self.contact_body_mask, strike_body_mask=self.strike_body_mask, progress_buf=progress_buf.data_ptr(),
            max_episode_length=self.max_episode_length, prev_root_pos=self._prev_root_pos.data_ptr(), dt=self.dt,
            obs_buf=self.obs_buf.data_ptr(), obs_stride=self.obs_buf.stride(0), rew_buf=self.rew_buf.data_ptr(), reset_buf=self.reset_buf.data_ptr(),
            terminate_buf=self._terminate_buf.data_ptr())

    def _launch(self, a) -> None:
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_ztask_step(C.byref(a), self.num_envs, _lib.current_stream(self.device)), "pulse_ztask_step")

    def _launch_list(self, a, env_list: torch.Tensor, count: torch.Tensor) -> None:
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_ztask_obs_list(C.byref(a), env_list.data_ptr(), count.data_ptr(), self.num_envs,
                                                     _lib.current_stream(self.device)), "pulse_ztask_obs_list")


class SpeedTaskB200(_ZTaskBase):
    """HumanoidSpeed (humanoid_speed.py:17-240): run along +x at a commanded speed."""
    kind, obs_size = _lib.ZTASK_SPEED, SPEED_OBS

    def __init__(self, num_envs: int, device="cuda:0", contact_bodies: Sequence[str] = ("R_Ankle", "L_Ankle", "R_Toe", "L_Toe"),
                 tar_speed_min: float = 0.0, tar_speed_max: float = 5.0, speed_change_steps_min: int = 100, speed_change_steps_max: int = 200,
                 max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15, dt: float = 1.0 / 30.0,
                 power_reward: bool = False, power_coefficient: float = 0.0005):
        super().__init__(num_envs, device, contact_bodies, max_episode_length, enable_early_termination, termination_height, dt)
        self._tar_speed_min, self._tar_speed_max = tar_speed_min, tar_speed_max
        self._speed_change_steps_min, self._speed_change_steps_max = speed_change_steps_min, speed_change_steps_max
        self.power_reward, self.power_coefficient = power_reward, power_coefficient
        dev = self.device
        self._tar_speed = torch.ones(num_envs, device=dev)                                    # :41
        self._speed_change_steps = torch.zeros(num_envs, dtype=torch.int64, device=dev)       # :39
        self.reward_raw = torch.zeros(num_envs, 2 if power_reward else 1, device=dev)

    def get_task_obs_size(self) -> int:
        return 3

    def update_task(self, progress_buf: torch.Tensor, rand01: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None) -> None:
        """_update_task / _reset_task (:157-175) without the `nonzero` host sync: every env draws, the envs whose progress reached
        `_speed_change_steps` take the draw (same distribution; the reference draws for the selected subset only)."""
        n, dev = self.num_envs, self.device
        rand01 = torch.rand(n, device=dev) if rand01 is None else rand01
        steps = torch.randint(self._speed_change_steps_min, self._speed_change_steps_max, (n,), device=dev) if steps is None else steps
        m = progress_buf >= self._speed_change_steps
        self._tar_speed.copy_(torch.where(m, (self._tar_speed_max - self._tar_speed_min) * rand01 + self._tar_speed_min, self._tar_speed))
        self._speed_change_steps.copy_(torch.where(m, progress_buf + steps, self._speed_change_steps))

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None, dof_vel: Optional[torch.Tensor] = None) -> None:
        """_compute_reward (:199-222) + _compute_reset (Humanoid's) + _compute_observations in one launch."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        a.tar_speed, a.reward_raw, a.raw_stride = self._tar_speed.data_ptr(), self.reward_raw.data_ptr(), self.reward_raw.stride(0)
        if self.power_reward:
            if dof_force is None or dof_vel is None:
                raise _lib.PulseError("power_reward needs dof_force and dof_vel")
            a.dof_force, a.dof_force_stride, a.power_coefficient = dof_force.data_ptr(), dof_force.stride(0), self.power_coefficient
            a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_vel.data_ptr(), dof_vel.stride(0), dof_vel.stride(1)
        self._launch(a)

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count): post_physics_step's rows for them, nothing else."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        a.tar_speed = self._tar_speed.data_ptr()
        self._launch_list(a, env_list, count)


class StrikeTaskB200(_ZTaskBase):
    """HumanoidStrike (humanoid_strike.py:17-240): walk to a standing target and knock it over."""
    kind, obs_size = _lib.ZTASK_STRIKE, STRIKE_OBS

    def __init__(self, num_envs: int, device="cuda:0", contact_bodies: Sequence[str] = ("R_Ankle", "L_Ankle", "R_Toe", "L_Toe"),
                 strike_bodies: Sequence[str] = ("R_Wrist", "R_Hand"), tar_dist_min: float = 0.5, tar_dist_max: float = 10.0, near_dist: float = 1.5,
                 near_prob: float = 0.5, max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15,
                 dt: float = 1.0 / 30.0):
        super().__init__(num_envs, device, contact_bodies, max_episode_length, enable_early_termination, termination_height, dt)
        self.strike_body_mask = _mask(strike_bodies)
        self._tar_dist_min, self._tar_dist_max, self._near_dist, self._near_prob = tar_dist_min, tar_dist_max, near_dist, near_prob

    def get_task_obs_size(self) -> int:
        return 15

    def reset_target(self, env_ids: torch.Tensor, root_states: torch.Tensor, target_states: torch.Tensor, rand: Optional[torch.Tensor] = None) -> None:
        """_reset_target (humanoid_strike.py:124-145): place the target at a random distance / bearing around the character, upright,
        random yaw, at rest.  `target_states` is the [N, 13] view of the target actor's root state, written in place; `rand` [n, 4]
        injects the four uniform draws (near, distance, bearing, yaw)."""
        n = int(env_ids.shape[0])
        if n == 0:
            return
        r = torch.rand(n, 4, device=self.device) if rand is None else rand
        dist_max = torch.where(r[:, 0] < self._near_prob, torch.full_like(r[:, 0], self._near_dist), torch.full_like(r[:, 0], self._tar_dist_max))
        dist = (dist_max - self._tar_dist_min) * r[:, 1] + self._tar_dist_min
        theta, yaw = 2 * math.pi * r[:, 2], 2 * math.pi * r[:, 3]
        target_states[env_ids, 0] = dist * torch.cos(theta) + root_states[env_ids, 0]
        target_states[env_ids, 1] = dist * torch.sin(theta) + root_states[env_ids, 1]
        target_states[env_ids, 2] = 0.9
        zero = torch.zeros_like(yaw)
        target_states[env_ids, 3:7] = torch.stack([zero, zero, torch.sin(0.5 * yaw), torch.cos(0.5 * yaw)], dim=-1)   # quat_from_angle_axis(yaw, z)
        target_states[env_ids, 7:13] = 0.0

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, target_states: torch.Tensor,
                          tar_contact_forces: torch.Tensor, contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_reward (:176-185) + _compute_reset (:201-207) + _compute_observations in one launch.  target_states [N, 13] and
        tar_contact_forces [N, 3] are views of the simulator tensors (:109, :116), read through their env strides."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        a.target_states, a.target_env_stride = target_states.data_ptr(), target_states.stride(0)
        a.tar_contact_forces, a.tar_contact_env_stride = tar_contact_forces.data_ptr(), tar_contact_forces.stride(0)
        self._launch(a)

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     target_states: torch.Tensor, contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count): post_physics_step's rows for them, nothing else."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        a.target_states, a.target_env_stride = target_states.data_ptr(), target_states.stride(0)
        self._launch_list(a, env_list, count)


class SmplxSpeedTaskB200:
    """HumanoidSpeed(Z) for the 52-body SMPL-X humanoid of PULSE-X (`env.task=HumanoidSpeedZ env=env_pulsex_amp robot=smplx_humanoid`):
    the post-physics step `pulse_smplx_speed_step` and `_update_task`.  The self observation takes the heading of
    remove_base_rot(root_rot) (has_upright_start False), the task observation that of the raw root rotation, as the reference does;
    obs = [self 778 | 3].  Bodies are given by index in the simulator's body order (SMPLH_MUJOCO_NAMES): `contact_body_ids` is the
    task's `_contact_body_ids` (R_Ankle, L_Ankle, R_Toe, L_Toe in env_pulsex_amp.yaml).  env_pulsex_amp.yaml has power_reward and
    power_usage_reward off; neither term is served, and a `dof_force` is refused."""
    kind, obs_size, layout = _lib.ZTASK_SPEED, _lib.SMPLX_SPEED_OBS, "smplx"

    def __init__(self, num_envs: int, device="cuda:0", *, contact_body_ids: Sequence[int], tar_speed_min: float = 0.0, tar_speed_max: float = 5.0,
                 speed_change_steps_min: int = 100, speed_change_steps_max: int = 200, max_episode_length: int = 300,
                 enable_early_termination: bool = True, termination_height: float = 0.15, dt: float = 1.0 / 30.0, power_reward: bool = False):
        if power_reward:
            raise _lib.PulseError("SmplxSpeedTaskB200: the power reward is not served for SMPL-X (env_pulsex_amp.yaml has power_reward False)")
        B = _lib.SMPLX_BODIES
        ids = [int(i) for i in contact_body_ids]
        if any(i < 0 or i >= B for i in ids):
            raise _lib.PulseError(f"SmplxSpeedTaskB200: contact_body_ids {ids} outside [0, {B})")
        self.device, self.num_envs = torch.device(device), int(num_envs)
        self.contact_body_mask = sum(1 << i for i in set(ids))
        self.max_episode_length, self.enable_early_termination, self.dt = int(max_episode_length), bool(enable_early_termination), float(dt)
        self._tar_speed_min, self._tar_speed_max = tar_speed_min, tar_speed_max
        self._speed_change_steps_min, self._speed_change_steps_max = speed_change_steps_min, speed_change_steps_max
        self.power_reward = False
        dev, n = self.device, self.num_envs
        self.termination_heights = torch.full((B,), termination_height, device=dev)
        self._prev_root_pos = torch.zeros(n, 3, device=dev)
        self._tar_speed = torch.ones(n, device=dev)
        self._speed_change_steps = torch.zeros(n, dtype=torch.int64, device=dev)
        self.obs_buf = torch.zeros(n, self.obs_size, device=dev)
        self.rew_buf = torch.zeros(n, device=dev)
        self.reward_raw = torch.zeros(n, 1, device=dev)
        self.reset_buf = torch.zeros(n, dtype=torch.int64, device=dev)
        self._terminate_buf = torch.zeros(n, dtype=torch.int64, device=dev)
        self.lib = _lib.load()

    def get_task_obs_size(self) -> int:
        return 3

    pre_physics_step = _ZTaskBase.pre_physics_step
    update_task = SpeedTaskB200.update_task

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        B = _lib.SMPLX_BODIES
        if rigid_body_state.dim() != 3 or rigid_body_state.shape[1] < B or rigid_body_state.stride(1) != 13 or rigid_body_state.stride(2) != 1:
            raise _lib.PulseError(f"rigid_body_state must be a [N, B>={B}, 13] view with row stride 13")
        if contact_forces is not None and (contact_forces.dim() != 3 or contact_forces.shape[1] < B or contact_forces.stride(1) != 3
                                           or contact_forces.stride(2) != 1):
            raise _lib.PulseError(f"contact_forces must be a [N, B>={B}, 3] view with contiguous bodies")
        return _lib.SmplxSpeedStepArgs(
            enable_early_termination=int(self.enable_early_termination), body_state=rigid_body_state.data_ptr(),
            body_env_stride=rigid_body_state.stride(0), contact_forces=contact_forces.data_ptr() if contact_forces is not None else None,
            contact_env_stride=contact_forces.stride(0) if contact_forces is not None else 0, termination_heights=self.termination_heights.data_ptr(),
            contact_body_mask=self.contact_body_mask, progress_buf=progress_buf.data_ptr(), max_episode_length=self.max_episode_length,
            prev_root_pos=self._prev_root_pos.data_ptr(), dt=self.dt, tar_speed=self._tar_speed.data_ptr(), obs_buf=self.obs_buf.data_ptr(),
            obs_stride=self.obs_buf.stride(0), rew_buf=self.rew_buf.data_ptr(), reward_raw=self.reward_raw.data_ptr(),
            raw_stride=self.reward_raw.stride(0), reset_buf=self.reset_buf.data_ptr(), terminate_buf=self._terminate_buf.data_ptr())

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None) -> None:
        """compute_speed_reward + compute_humanoid_reset + the observation in one launch."""
        if dof_force is not None:
            raise _lib.PulseError("SmplxSpeedTaskB200: dof_force given, but the SMPL-X speed step has no power term")
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_smplx_speed_step(C.byref(a), self.num_envs, _lib.current_stream(self.device)), "pulse_smplx_speed_step")

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count): post_physics_step's rows for them, nothing else."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_smplx_speed_obs_list(C.byref(a), env_list.data_ptr(), count.data_ptr(), self.num_envs,
                                                           _lib.current_stream(self.device)), "pulse_smplx_speed_obs_list")


def _smplx_body_mask(who: str, name: str, ids: Sequence[int]) -> int:
    B = _lib.SMPLX_BODIES
    ids = [int(i) for i in ids]
    if any(i < 0 or i >= B for i in ids):
        raise _lib.PulseError(f"{who}: {name} {ids} outside [0, {B})")
    return sum(1 << i for i in set(ids))


class _SmplxTargetTask:
    """The state and launches the SMPL-X reach and strike step objects share (`pulse_smplx_target_step` and its list observation)."""
    kind, obs_size, layout = 0, 0, "smplx"

    def __init__(self, who: str, num_envs: int, device, contact_body_ids, max_episode_length: int, enable_early_termination: bool,
                 termination_height: float, power_reward: bool, power_usage_reward: bool):
        if power_reward or power_usage_reward:
            raise _lib.PulseError(f"{who}: power_reward / power_usage_reward are not served for SMPL-X (env_pulsex_amp.yaml has both off)")
        self.who = who
        self.contact_body_mask = _smplx_body_mask(who, "contact_body_ids", contact_body_ids)
        self.strike_body_mask, self.reach_body_id = 0, 0
        self.device, self.num_envs = torch.device(device), int(num_envs)
        self.max_episode_length, self.enable_early_termination = int(max_episode_length), bool(enable_early_termination)
        self.power_reward = False
        dev, n = self.device, self.num_envs
        self.termination_heights = torch.full((_lib.SMPLX_BODIES,), termination_height, device=dev)
        self.obs_buf = torch.zeros(n, self.obs_size, device=dev)
        self.rew_buf = torch.zeros(n, device=dev)
        self.reset_buf = torch.zeros(n, dtype=torch.int64, device=dev)
        self._terminate_buf = torch.zeros(n, dtype=torch.int64, device=dev)
        self.lib = _lib.load()

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        """The step arguments without the task's target views (the strike task adds them)."""
        B = _lib.SMPLX_BODIES
        if rigid_body_state.dim() != 3 or rigid_body_state.shape[1] < B or rigid_body_state.stride(1) != 13 or rigid_body_state.stride(2) != 1:
            raise _lib.PulseError(f"rigid_body_state must be a [N, B>={B}, 13] view with row stride 13")
        if contact_forces is not None and (contact_forces.dim() != 3 or contact_forces.shape[1] < B or contact_forces.stride(1) != 3
                                           or contact_forces.stride(2) != 1):
            raise _lib.PulseError(f"contact_forces must be a [N, B>={B}, 3] view with contiguous bodies")
        return _lib.SmplxTargetStepArgs(
            kind=self.kind, enable_early_termination=int(self.enable_early_termination), body_state=rigid_body_state.data_ptr(),
            body_env_stride=rigid_body_state.stride(0), contact_forces=contact_forces.data_ptr() if contact_forces is not None else None,
            contact_env_stride=contact_forces.stride(0) if contact_forces is not None else 0, termination_heights=self.termination_heights.data_ptr(),
            contact_body_mask=self.contact_body_mask, strike_body_mask=self.strike_body_mask, reach_body_id=self.reach_body_id,
            progress_buf=progress_buf.data_ptr(), max_episode_length=self.max_episode_length, obs_buf=self.obs_buf.data_ptr(),
            obs_stride=self.obs_buf.stride(0), rew_buf=self.rew_buf.data_ptr(), reset_buf=self.reset_buf.data_ptr(),
            terminate_buf=self._terminate_buf.data_ptr())

    def _launch(self, a, dof_force) -> None:
        if dof_force is not None:
            raise _lib.PulseError(f"{self.who}: dof_force given, but the SMPL-X {_KIND_NAMES[self.kind]} step has no power term")
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_smplx_target_step(C.byref(a), self.num_envs, _lib.current_stream(self.device)), "pulse_smplx_target_step")

    def _launch_list(self, a, env_list: torch.Tensor, count: torch.Tensor) -> None:
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_smplx_target_obs_list(C.byref(a), env_list.data_ptr(), count.data_ptr(), self.num_envs,
                                                            _lib.current_stream(self.device)), "pulse_smplx_target_obs_list")


_KIND_NAMES = {_lib.ZTASK_REACH: "reach", _lib.ZTASK_STRIKE: "strike"}


class SmplxReachTaskB200(_SmplxTargetTask):
    """HumanoidReach(Z) for the 52-body SMPL-X humanoid of PULSE-X (`env.task=HumanoidReachZ env=env_pulsex_amp robot=smplx_humanoid`):
    the post-physics step `pulse_smplx_target_step` and `_update_task`, with what ReachTaskB200 carries.  The self observation takes the
    heading of remove_base_rot(root_rot), the target offset that of the raw root rotation, as the reference does; obs = [self 778 | 3].
    Bodies are indices in the simulator's body order (SMPLH_MUJOCO_NAMES): `reach_body_id` is `_reach_body_id`, `contact_body_ids` the
    task's `_contact_body_ids`.  The SMPL-X humanoid has no R_Hand body; its right arm is R_Elbow 35, R_Wrist 36 and the finger bodies
    37-51.  power_reward / power_usage_reward are refused, as is a `dof_force`."""
    kind, obs_size = _lib.ZTASK_REACH, _lib.SMPLX_REACH_OBS

    def __init__(self, num_envs: int, device="cuda:0", *, reach_body_id: int, contact_body_ids: Sequence[int], tar_change_steps_min: int = 100,
                 tar_change_steps_max: int = 200, tar_dist_max: float = 1.0, tar_height_min: float = 0.5, tar_height_max: float = 1.5,
                 max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15,
                 power_reward: bool = False, power_usage_reward: bool = False):
        _smplx_body_mask("SmplxReachTaskB200", "reach_body_id", [reach_body_id])
        super().__init__("SmplxReachTaskB200", num_envs, device, contact_body_ids, max_episode_length, enable_early_termination,
                         termination_height, power_reward, power_usage_reward)
        self.reach_body_id = int(reach_body_id)
        self.tar_change_steps_min, self.tar_change_steps_max = tar_change_steps_min, tar_change_steps_max
        self.tar_dist_max, self.tar_height_min, self.tar_height_max = tar_dist_max, tar_height_min, tar_height_max
        dev, n = self.device, self.num_envs
        self._tar_pos = torch.zeros(n, 3, device=dev)
        self._tar_change_steps = torch.zeros(n, dtype=torch.int64, device=dev)
        self._rand = torch.zeros(n, 3, device=dev)
        self._steps = torch.zeros(n, dtype=torch.int64, device=dev)

    def get_task_obs_size(self) -> int:
        return 3

    update_task = ReachTaskB200.update_task     # pulse_reach_update_task does not depend on the body layout

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        a = super()._args(rigid_body_state, progress_buf, contact_forces)
        a.tar_pos = self._tar_pos.data_ptr()
        return a

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None) -> None:
        """compute_reach_reward + compute_humanoid_reset + the observation in one launch."""
        self._launch(self._args(rigid_body_state, progress_buf, contact_forces), dof_force)

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count): post_physics_step's rows for them, nothing else."""
        self._launch_list(self._args(rigid_body_state, progress_buf, contact_forces), env_list, count)


class SmplxStrikeTaskB200(_SmplxTargetTask):
    """HumanoidStrike(Z) for the 52-body SMPL-X humanoid of PULSE-X (`env.task=HumanoidStrikeZ env=env_pulsex_amp robot=smplx_humanoid`):
    the post-physics step `pulse_smplx_target_step`, with what StrikeTaskB200 carries.  obs = [self 778 | 15], the target in the heading
    of the raw root rotation.  `strike_body_ids` is `_strike_body_ids`, `contact_body_ids` `_contact_body_ids`, both indices in the
    simulator's body order (SMPL-X has no R_Hand; the right arm is R_Elbow 35, R_Wrist 36 and the finger bodies 37-51).  The early
    termination's pushing body is any body outside both sets pressing harder than 50 N, over all 52 bodies.  power_reward /
    power_usage_reward are refused, as is a `dof_force`."""
    kind, obs_size = _lib.ZTASK_STRIKE, _lib.SMPLX_STRIKE_OBS

    def __init__(self, num_envs: int, device="cuda:0", *, strike_body_ids: Sequence[int], contact_body_ids: Sequence[int],
                 tar_dist_min: float = 0.5, tar_dist_max: float = 10.0, near_dist: float = 1.5, near_prob: float = 0.5,
                 max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15, dt: float = 1.0 / 30.0,
                 power_reward: bool = False, power_usage_reward: bool = False):
        strike_mask = _smplx_body_mask("SmplxStrikeTaskB200", "strike_body_ids", strike_body_ids)
        super().__init__("SmplxStrikeTaskB200", num_envs, device, contact_body_ids, max_episode_length, enable_early_termination,
                         termination_height, power_reward, power_usage_reward)
        self.strike_body_mask, self.dt = strike_mask, float(dt)
        self._tar_dist_min, self._tar_dist_max, self._near_dist, self._near_prob = tar_dist_min, tar_dist_max, near_dist, near_prob
        self._prev_root_pos = torch.zeros(self.num_envs, 3, device=self.device)

    def get_task_obs_size(self) -> int:
        return 15

    pre_physics_step = _ZTaskBase.pre_physics_step
    reset_target = StrikeTaskB200.reset_target

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        a = super()._args(rigid_body_state, progress_buf, contact_forces)
        a.prev_root_pos, a.dt = self._prev_root_pos.data_ptr(), self.dt
        return a

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, target_states: torch.Tensor,
                          tar_contact_forces: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None) -> None:
        """compute_strike_reward + the strike compute_humanoid_reset + the observation in one launch.  target_states [N, 13] and
        tar_contact_forces [N, 3] are views of the simulator tensors, read through their env strides."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        a.target_states, a.target_env_stride = target_states.data_ptr(), target_states.stride(0)
        a.tar_contact_forces, a.tar_contact_env_stride = tar_contact_forces.data_ptr(), tar_contact_forces.stride(0)
        self._launch(a, dof_force)

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     target_states: torch.Tensor, contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count): post_physics_step's rows for them, nothing else."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        a.target_states, a.target_env_stride = target_states.data_ptr(), target_states.stride(0)
        self._launch_list(a, env_list, count)
