"""Downstream latent-space reach, speed and strike tasks (SURVEY K21, 8f-4): host-side mirrors of `HumanoidReach(Z)` /
`HumanoidSpeed(Z)` / `HumanoidStrike(Z)` (phc/env/tasks/humanoid_reach.py, humanoid_speed.py, humanoid_strike.py) for the post-physics
path -- reward, reset, observation in ONE launch -- and the task-state updates (`_update_task` / `_reset_task`).  The policy acts in the
frozen PULSE latent space: `HumanoidZ.step -> step_z` decodes the action through the prior + decoder (`PulseVAE.compute_z_actions`)
before `pre_physics_step` maps it to PD targets (`pulse_b200.vae.pd_targets`).  Isaac Gym keeps the physics and owns the state tensors,
which are read in place.
`ReachTaskB200`, `SpeedTaskB200` and `StrikeTaskB200` serve the 24-body SMPL humanoid (`pulse_reach_step`, `pulse_ztask_step`);
`SmplxReachTaskB200`, `SmplxSpeedTaskB200` and `SmplxStrikeTaskB200`, each a subclass of its SMPL counterpart, the 52-body SMPL-X
humanoid of PULSE-X (`pulse_smplx_target_step`, `pulse_smplx_speed_step`).
"""
import ctypes as C
import math
from typing import Optional, Sequence

import torch

from . import _lib

REACH_OBS = 361                       # 358 self observation + 3 (target offset in the heading frame), humanoid_reach.py:69-74
SPEED_OBS, STRIKE_OBS = 361, 373      # 358 self observation + 3 / + 15
# SMPL humanoid body order (smpl_humanoid.xml); contact bodies of the reach configs = both ankles and toes
SMPL_BODY_NAMES = ['Pelvis', 'L_Hip', 'L_Knee', 'L_Ankle', 'L_Toe', 'R_Hip', 'R_Knee', 'R_Ankle', 'R_Toe', 'Torso', 'Spine', 'Chest', 'Neck',
                   'Head', 'L_Thorax', 'L_Shoulder', 'L_Elbow', 'L_Wrist', 'L_Hand', 'R_Thorax', 'R_Shoulder', 'R_Elbow', 'R_Wrist', 'R_Hand']
_SMPLX_TARGET_ENTRIES = ("pulse_smplx_target_step", "pulse_smplx_target_obs_list", "pulse_smplx_target_rollout_step")
_ZTASK_ENTRIES = ("pulse_ztask_step", "pulse_ztask_obs_list", "pulse_ztask_rollout_step")


def _no_power_reward(who: str, power_reward: bool, power_usage_reward: bool = False) -> None:
    if power_reward or power_usage_reward:
        raise _lib.PulseError(f"{who}: power_reward / power_usage_reward are not served for SMPL-X (env_pulsex_amp.yaml has both off)")


def _no_dof_force(task, dof_force) -> None:
    if dof_force is not None:
        raise _lib.PulseError(f"{type(task).__name__}: dof_force given, but the SMPL-X steps have no power term")


class _TaskStep:
    """What every latent-task step object holds: the body masks, the termination heights, the step's output buffers, its argument
    struct (`_args`) and the launches of its entry points.  `layout` "smpl": 24 bodies, body sets given by name (SMPL_BODY_NAMES);
    "smplx": 52 bodies, body sets given by index in the simulator's body order (SMPLH_MUJOCO_NAMES).  `Args` is the argument struct,
    `entries` its (step, list observation, rollout step) entry points."""
    kind, obs_size = 0, 0
    layout, bodies, Args, entries = "smpl", 24, None, ()
    power_reward = False

    def __init__(self, num_envs: int, device, contact_bodies, max_episode_length: int, enable_early_termination: bool,
                 termination_height: float):
        self.device, self.num_envs = torch.device(device), int(num_envs)
        self.contact_body_mask = self._body_mask("contact_body_ids", contact_bodies)
        self.max_episode_length, self.enable_early_termination = int(max_episode_length), bool(enable_early_termination)
        dev, n = self.device, self.num_envs
        self.termination_heights = torch.full((self.bodies,), termination_height, device=dev)
        self.obs_buf = torch.zeros(n, self.obs_size, device=dev)
        self.rew_buf = torch.zeros(n, device=dev)
        self.reset_buf = torch.zeros(n, dtype=torch.int64, device=dev)
        self._terminate_buf = torch.zeros(n, dtype=torch.int64, device=dev)
        self.lib = _lib.load()

    def _body_mask(self, what: str, bodies: Sequence) -> int:
        if self.layout == "smpl":
            return sum(1 << SMPL_BODY_NAMES.index(b) for b in set(bodies))
        ids = [int(i) for i in bodies]
        if any(i < 0 or i >= self.bodies for i in ids):
            raise _lib.PulseError(f"{type(self).__name__}: {what} {ids} outside [0, {self.bodies})")
        return sum(1 << i for i in set(ids))

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        """The step arguments over the simulator's views with this object's outputs; subclasses add their targets."""
        B = self.bodies
        if rigid_body_state.dim() != 3 or rigid_body_state.shape[1] < B or rigid_body_state.stride(1) != 13 or rigid_body_state.stride(2) != 1:
            raise _lib.PulseError(f"rigid_body_state must be a [N, B>={B}, 13] view with row stride 13")
        if contact_forces is not None and (contact_forces.dim() != 3 or contact_forces.shape[1] < B or contact_forces.stride(1) != 3
                                           or contact_forces.stride(2) != 1):
            raise _lib.PulseError(f"contact_forces must be a [N, B>={B}, 3] view with contiguous bodies")
        a = self.Args(
            enable_early_termination=int(self.enable_early_termination), body_state=rigid_body_state.data_ptr(),
            body_env_stride=rigid_body_state.stride(0), contact_forces=contact_forces.data_ptr() if contact_forces is not None else None,
            contact_env_stride=contact_forces.stride(0) if contact_forces is not None else 0, termination_heights=self.termination_heights.data_ptr(),
            contact_body_mask=self.contact_body_mask, progress_buf=progress_buf.data_ptr(), max_episode_length=self.max_episode_length,
            obs_buf=self.obs_buf.data_ptr(), obs_stride=self.obs_buf.stride(0), rew_buf=self.rew_buf.data_ptr(), reset_buf=self.reset_buf.data_ptr(),
            terminate_buf=self._terminate_buf.data_ptr())
        if hasattr(self.Args, "kind"):      # the structs that serve more than one task kind
            a.kind = self.kind
        return a

    def _launch(self, a) -> None:
        with torch.cuda.device(self.device):
            _lib.check(getattr(self.lib, self.entries[0])(C.byref(a), self.num_envs, _lib.current_stream(self.device)), self.entries[0])

    def _launch_list(self, a, env_list: torch.Tensor, count: torch.Tensor) -> None:
        with torch.cuda.device(self.device):
            _lib.check(getattr(self.lib, self.entries[1])(C.byref(a), env_list.data_ptr(), count.data_ptr(), self.num_envs,
                                                          _lib.current_stream(self.device)), self.entries[1])


class _RootVelocityTaskStep(_TaskStep):
    """The speed and strike tasks: their rewards read the root velocity as the root's displacement over the physics step, dt."""

    def __init__(self, num_envs: int, device, contact_bodies, max_episode_length: int, enable_early_termination: bool,
                 termination_height: float, dt: float):
        super().__init__(num_envs, device, contact_bodies, max_episode_length, enable_early_termination, termination_height)
        self.dt = float(dt)
        self._prev_root_pos = torch.zeros(self.num_envs, 3, device=self.device)

    def pre_physics_step(self, root_states: torch.Tensor) -> None:
        """`self._prev_root_pos[:] = self._humanoid_root_states[..., 0:3]` (humanoid_speed.py:73-76, humanoid_strike.py pre_physics_step)."""
        self._prev_root_pos.copy_(root_states[:, 0:3])

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        a = super()._args(rigid_body_state, progress_buf, contact_forces)
        a.prev_root_pos, a.dt = self._prev_root_pos.data_ptr(), self.dt
        return a


class ReachTaskB200(_TaskStep):
    """HumanoidReach (humanoid_reach.py:17-166, :224-250): bring one body to a target point resampled every 100-200 steps."""
    kind, obs_size = _lib.ZTASK_REACH, REACH_OBS
    Args, entries = _lib.ReachStepArgs, ("pulse_reach_step", "pulse_reach_obs_list", "pulse_reach_rollout_step")

    def __init__(self, num_envs: int, device="cuda:0", reach_body_name: str = "R_Hand", contact_bodies: Sequence[str] = ("R_Ankle", "L_Ankle", "R_Toe", "L_Toe"),
                 tar_change_steps_min: int = 100, tar_change_steps_max: int = 200, tar_dist_max: float = 1.0, tar_height_min: float = 0.5,
                 tar_height_max: float = 1.5, max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15):
        super().__init__(num_envs, device, contact_bodies, max_episode_length, enable_early_termination, termination_height)
        self._body_mask("reach_body_id", [reach_body_name])
        self.reach_body_id = SMPL_BODY_NAMES.index(reach_body_name) if self.layout == "smpl" else int(reach_body_name)
        self.tar_change_steps_min, self.tar_change_steps_max = tar_change_steps_min, tar_change_steps_max
        self.tar_dist_max, self.tar_height_min, self.tar_height_max = tar_dist_max, tar_height_min, tar_height_max
        dev, n = self.device, self.num_envs
        self._tar_pos = torch.zeros(n, 3, device=dev)
        self._tar_change_steps = torch.zeros(n, dtype=torch.int64, device=dev)
        self._rand = torch.zeros(n, 3, device=dev)
        self._steps = torch.zeros(n, dtype=torch.int64, device=dev)

    def get_task_obs_size(self) -> int:
        return 3

    def update_task(self, progress_buf: torch.Tensor, rand01: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None) -> None:
        """_update_task (:126-131): resample the target of every env whose progress reached `_tar_change_steps`.
        The uniform draws can be injected (tests); by default they are drawn for all envs on the device (the reference draws
        only for the selected subset -- same distribution, different random stream).  pulse_reach_update_task does not depend on the
        body layout."""
        if rand01 is None:
            rand01 = self._rand.uniform_()
        if steps is None:
            steps = self._steps.random_(self.tar_change_steps_min, self.tar_change_steps_max)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_reach_update_task(progress_buf.data_ptr(), self._tar_change_steps.data_ptr(), self._tar_pos.data_ptr(),
                                                        rand01.data_ptr(), steps.data_ptr(), self.tar_dist_max, self.tar_height_min, self.tar_height_max,
                                                        self.num_envs, _lib.current_stream(self.device)), "pulse_reach_update_task")

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        a = super()._args(rigid_body_state, progress_buf, contact_forces)
        a.tar_pos, a.reach_body_id = self._tar_pos.data_ptr(), self.reach_body_id
        return a

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_reward + _compute_reset + _compute_observations (humanoid.py:1315-1330 order) in one launch.
        rigid_body_state fp32 [N, B_env >= 24, 13] (Isaac Gym view, read in place); contact_forces fp32 [N, B_env, 3]."""
        self._launch(self._args(rigid_body_state, progress_buf, contact_forces))

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count) (int64 list, int32 device-side count): the rows
        post_physics_step writes for them, bit for bit, and nothing else."""
        self._launch_list(self._args(rigid_body_state, progress_buf, contact_forces), env_list, count)


class SpeedTaskB200(_RootVelocityTaskStep):
    """HumanoidSpeed (humanoid_speed.py:17-240): run along +x at a commanded speed."""
    kind, obs_size = _lib.ZTASK_SPEED, SPEED_OBS
    Args, entries = _lib.ZTaskStepArgs, _ZTASK_ENTRIES

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

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        a = super()._args(rigid_body_state, progress_buf, contact_forces)
        a.tar_speed, a.reward_raw, a.raw_stride = self._tar_speed.data_ptr(), self.reward_raw.data_ptr(), self.reward_raw.stride(0)
        return a

    def _power_args(self, a, dof_force: Optional[torch.Tensor], dof_vel: Optional[torch.Tensor]) -> None:
        """The power term's inputs (:215-222) into the step arguments `a` when power_reward is on."""
        if not self.power_reward:
            return
        if dof_force is None or dof_vel is None:
            raise _lib.PulseError("power_reward needs dof_force and dof_vel")
        a.dof_force, a.dof_force_stride, a.power_coefficient = dof_force.data_ptr(), dof_force.stride(0), self.power_coefficient
        a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_vel.data_ptr(), dof_vel.stride(0), dof_vel.stride(1)

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None, dof_vel: Optional[torch.Tensor] = None) -> None:
        """_compute_reward (:199-222) + _compute_reset (Humanoid's) + _compute_observations in one launch."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        self._power_args(a, dof_force, dof_vel)
        self._launch(a)

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count): post_physics_step's rows for them, nothing else."""
        self._launch_list(self._args(rigid_body_state, progress_buf, contact_forces), env_list, count)


class StrikeTaskB200(_RootVelocityTaskStep):
    """HumanoidStrike (humanoid_strike.py:17-240): walk to a standing target and knock it over."""
    kind, obs_size = _lib.ZTASK_STRIKE, STRIKE_OBS
    Args, entries = _lib.ZTaskStepArgs, _ZTASK_ENTRIES

    def __init__(self, num_envs: int, device="cuda:0", contact_bodies: Sequence[str] = ("R_Ankle", "L_Ankle", "R_Toe", "L_Toe"),
                 strike_bodies: Sequence[str] = ("R_Wrist", "R_Hand"), tar_dist_min: float = 0.5, tar_dist_max: float = 10.0, near_dist: float = 1.5,
                 near_prob: float = 0.5, max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15,
                 dt: float = 1.0 / 30.0):
        super().__init__(num_envs, device, contact_bodies, max_episode_length, enable_early_termination, termination_height, dt)
        self.strike_body_mask = self._body_mask("strike_body_ids", strike_bodies)
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

    def _args(self, rigid_body_state, progress_buf, contact_forces):
        a = super()._args(rigid_body_state, progress_buf, contact_forces)
        a.strike_body_mask = self.strike_body_mask
        return a

    @staticmethod
    def _target_args(a, target_states: torch.Tensor, tar_contact_forces: Optional[torch.Tensor] = None) -> None:
        """The target's views into the step arguments `a`: target_states [N, 13] and tar_contact_forces [N, 3] (:109, :116), read
        through their env strides; the list observation reads no contact."""
        a.target_states, a.target_env_stride = target_states.data_ptr(), target_states.stride(0)
        if tar_contact_forces is not None:
            a.tar_contact_forces, a.tar_contact_env_stride = tar_contact_forces.data_ptr(), tar_contact_forces.stride(0)

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, target_states: torch.Tensor,
                          tar_contact_forces: torch.Tensor, contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_reward (:176-185) + _compute_reset (:201-207) + _compute_observations in one launch."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        self._target_args(a, target_states, tar_contact_forces)
        self._launch(a)

    def observe_list(self, rigid_body_state: torch.Tensor, env_list: torch.Tensor, count: torch.Tensor, progress_buf: torch.Tensor,
                     target_states: torch.Tensor, contact_forces: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids) for the envs env_list[0 .. *count): post_physics_step's rows for them, nothing else."""
        a = self._args(rigid_body_state, progress_buf, contact_forces)
        self._target_args(a, target_states)
        self._launch_list(a, env_list, count)


class SmplxReachTaskB200(ReachTaskB200):
    """HumanoidReach(Z) for the 52-body SMPL-X humanoid of PULSE-X (`env.task=HumanoidReachZ env=env_pulsex_amp robot=smplx_humanoid`):
    the post-physics step `pulse_smplx_target_step` and `_update_task`, with what ReachTaskB200 carries.  The self observation takes the
    heading of remove_base_rot(root_rot), the target offset that of the raw root rotation, as the reference does; obs = [self 778 | 3].
    Bodies are indices in the simulator's body order (SMPLH_MUJOCO_NAMES): `reach_body_id` is `_reach_body_id`, `contact_body_ids` the
    task's `_contact_body_ids`.  The SMPL-X humanoid has no R_Hand body; its right arm is R_Elbow 35, R_Wrist 36 and the finger bodies
    37-51.  power_reward / power_usage_reward are refused, as is a `dof_force`."""
    obs_size, layout, bodies = _lib.SMPLX_REACH_OBS, "smplx", _lib.SMPLX_BODIES
    Args, entries = _lib.SmplxTargetStepArgs, _SMPLX_TARGET_ENTRIES

    def __init__(self, num_envs: int, device="cuda:0", *, reach_body_id: int, contact_body_ids: Sequence[int], tar_change_steps_min: int = 100,
                 tar_change_steps_max: int = 200, tar_dist_max: float = 1.0, tar_height_min: float = 0.5, tar_height_max: float = 1.5,
                 max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15,
                 power_reward: bool = False, power_usage_reward: bool = False):
        _no_power_reward("SmplxReachTaskB200", power_reward, power_usage_reward)
        super().__init__(num_envs, device, reach_body_id, contact_body_ids, tar_change_steps_min, tar_change_steps_max, tar_dist_max,
                         tar_height_min, tar_height_max, max_episode_length, enable_early_termination, termination_height)

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None) -> None:
        """compute_reach_reward + compute_humanoid_reset + the observation in one launch."""
        _no_dof_force(self, dof_force)
        super().post_physics_step(rigid_body_state, progress_buf, contact_forces)


class SmplxSpeedTaskB200(SpeedTaskB200):
    """HumanoidSpeed(Z) for the 52-body SMPL-X humanoid of PULSE-X (`env.task=HumanoidSpeedZ env=env_pulsex_amp robot=smplx_humanoid`):
    the post-physics step `pulse_smplx_speed_step` and `_update_task`.  The self observation takes the heading of
    remove_base_rot(root_rot) (has_upright_start False), the task observation that of the raw root rotation, as the reference does;
    obs = [self 778 | 3].  Bodies are given by index in the simulator's body order (SMPLH_MUJOCO_NAMES): `contact_body_ids` is the
    task's `_contact_body_ids` (R_Ankle, L_Ankle, R_Toe, L_Toe in env_pulsex_amp.yaml).  env_pulsex_amp.yaml has power_reward and
    power_usage_reward off; neither term is served, and a `dof_force` is refused."""
    obs_size, layout, bodies = _lib.SMPLX_SPEED_OBS, "smplx", _lib.SMPLX_BODIES
    Args, entries = _lib.SmplxSpeedStepArgs, ("pulse_smplx_speed_step", "pulse_smplx_speed_obs_list", "pulse_smplx_speed_rollout_step")

    def __init__(self, num_envs: int, device="cuda:0", *, contact_body_ids: Sequence[int], tar_speed_min: float = 0.0, tar_speed_max: float = 5.0,
                 speed_change_steps_min: int = 100, speed_change_steps_max: int = 200, max_episode_length: int = 300,
                 enable_early_termination: bool = True, termination_height: float = 0.15, dt: float = 1.0 / 30.0, power_reward: bool = False):
        _no_power_reward("SmplxSpeedTaskB200", power_reward)
        super().__init__(num_envs, device, contact_body_ids, tar_speed_min, tar_speed_max, speed_change_steps_min, speed_change_steps_max,
                         max_episode_length, enable_early_termination, termination_height, dt)

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None) -> None:
        """compute_speed_reward + compute_humanoid_reset + the observation in one launch."""
        _no_dof_force(self, dof_force)
        super().post_physics_step(rigid_body_state, progress_buf, contact_forces)


class SmplxStrikeTaskB200(StrikeTaskB200):
    """HumanoidStrike(Z) for the 52-body SMPL-X humanoid of PULSE-X (`env.task=HumanoidStrikeZ env=env_pulsex_amp robot=smplx_humanoid`):
    the post-physics step `pulse_smplx_target_step`, with what StrikeTaskB200 carries.  obs = [self 778 | 15], the target in the heading
    of the raw root rotation.  `strike_body_ids` is `_strike_body_ids`, `contact_body_ids` `_contact_body_ids`, both indices in the
    simulator's body order (SMPL-X has no R_Hand; the right arm is R_Elbow 35, R_Wrist 36 and the finger bodies 37-51).  The early
    termination's pushing body is any body outside both sets pressing harder than 50 N, over all 52 bodies.  power_reward /
    power_usage_reward are refused, as is a `dof_force`."""
    obs_size, layout, bodies = _lib.SMPLX_STRIKE_OBS, "smplx", _lib.SMPLX_BODIES
    Args, entries = _lib.SmplxTargetStepArgs, _SMPLX_TARGET_ENTRIES

    def __init__(self, num_envs: int, device="cuda:0", *, strike_body_ids: Sequence[int], contact_body_ids: Sequence[int],
                 tar_dist_min: float = 0.5, tar_dist_max: float = 10.0, near_dist: float = 1.5, near_prob: float = 0.5,
                 max_episode_length: int = 300, enable_early_termination: bool = True, termination_height: float = 0.15, dt: float = 1.0 / 30.0,
                 power_reward: bool = False, power_usage_reward: bool = False):
        _no_power_reward("SmplxStrikeTaskB200", power_reward, power_usage_reward)
        super().__init__(num_envs, device, contact_body_ids, strike_body_ids, tar_dist_min, tar_dist_max, near_dist, near_prob,
                         max_episode_length, enable_early_termination, termination_height, dt)

    def post_physics_step(self, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, target_states: torch.Tensor,
                          tar_contact_forces: torch.Tensor, contact_forces: Optional[torch.Tensor] = None,
                          dof_force: Optional[torch.Tensor] = None) -> None:
        """compute_strike_reward + the strike compute_humanoid_reset + the observation in one launch."""
        _no_dof_force(self, dof_force)
        super().post_physics_step(rigid_body_state, progress_buf, target_states, tar_contact_forces, contact_forces)
