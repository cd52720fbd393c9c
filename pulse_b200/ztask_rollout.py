"""The latent-space tasks' training iteration on the device (BASELINE config C5): the rollout of HumanoidReachZ / HumanoidSpeedZ /
HumanoidStrikeZ with the frozen PULSE prior + decoder, device resets and the latent policy's PPO update (`AMPAgent.play_steps` +
`train_epoch`, phc/learning/amp_agent.py:341-439; `HumanoidAMPTask` resets, humanoid_amp_task.py:57-76; `HumanoidZ.step -> step_z`,
humanoid_z.py:157-173; pulse_z_task.yaml)."""
import ctypes as C
from typing import Optional

import torch

from . import _lib
from .latent_rollout import LatentStepsB200

_KINDS = {_lib.ZTASK_REACH: "reach", _lib.ZTASK_SPEED: "speed", _lib.ZTASK_STRIKE: "strike"}
# the observation width per (body layout, task kind)
_WIDTHS = {("smpl", "reach"): 361, ("smpl", "speed"): 361, ("smpl", "strike"): 373, ("smplx", "reach"): _lib.SMPLX_REACH_OBS,
           ("smplx", "speed"): _lib.SMPLX_SPEED_OBS, ("smplx", "strike"): _lib.SMPLX_STRIKE_OBS}
# per body layout: (self observation -> dof targets of the decoder, latent size or None = any)
_LAYOUTS = {"smpl": (358, 69, None), "smplx": (_lib.SMPLX_SELF_OBS, _lib.SMPLX_DOF, 48)}
SIM_KEYS = ("body_state", "root_states", "dof_pos", "dof_vel", "progress_buf", "sampled_motion_ids", "motion_start_times")
STRIKE_KEYS = ("target_states", "tar_contact_forces")


def check_pieces(task, reset, policy, vae, amp=None) -> str:
    """The task kind ("reach" / "speed" / "strike") after checking that the step object, the reset, the latent policy and the frozen
    VAE belong together; raises PulseError otherwise.  SMPL: observations of 361 / 361 / 373 floats, a 358 -> 69 decoder.  SMPL-X
    (SmplxReachTaskB200 / SmplxSpeedTaskB200 / SmplxStrikeTaskB200, PULSE-X): 781 / 781 / 793 floats, a 778 -> 153 decoder and a
    48-dimensional latent (env_pulsex_amp.yaml).  `vae=None`: the dof-space baseline (learning=ppo), whose policy acts in the
    layout's 69 / 153 dofs."""
    kind = _KINDS.get(getattr(task, "kind", None))
    if kind is None:
        raise _lib.PulseError("ZTaskStepsB200: task must be a ReachTaskB200, SpeedTaskB200, StrikeTaskB200 or one of their SMPL-X "
                              "counterparts (SmplxReachTaskB200, SmplxSpeedTaskB200, SmplxStrikeTaskB200)")
    if getattr(reset, "kind", None) != kind:
        raise _lib.PulseError(f"ZTaskStepsB200: the reset serves {getattr(reset, 'kind', None)!r}, the task is {kind!r}")
    layout = getattr(task, "layout", "smpl")
    if bool(getattr(reset, "smplx", False)) != (layout == "smplx"):
        raise _lib.PulseError(f"ZTaskStepsB200: the task is {layout}, the reset's MotionLib has {getattr(reset, 'bodies', 24)} bodies")
    S, A, E = _LAYOUTS[layout]
    W = _WIDTHS[(layout, kind)]
    if int(task.obs_size) != W or int(policy.obs_size) != W:
        raise _lib.PulseError(f"ZTaskStepsB200: the {layout} {kind} observation has {W} floats, the task writes {task.obs_size} and the policy reads {policy.obs_size}")
    if vae is None:
        if int(policy.A) != A:
            raise _lib.PulseError(f"ZTaskStepsB200: without a VAE the policy acts in the {layout} humanoid's {A} dofs, not in {policy.A} "
                                  f"dimensions (a latent-space policy needs its VAE)")
    else:
        if int(policy.A) == A:
            raise _lib.PulseError(f"ZTaskStepsB200: the policy acts in the {layout} humanoid's {A} dofs, but a VAE was given (the "
                                  f"dof-space baseline takes vae=None)")
        if int(policy.A) != int(vae.E):
            raise _lib.PulseError(f"ZTaskStepsB200: the policy acts in {policy.A} dimensions, the VAE's latent has {vae.E}")
        if int(vae.S) != S or int(vae.A) != A:
            raise _lib.PulseError(f"ZTaskStepsB200: the decoder must map the {S}-float self observation to {A} dof targets, not {vae.S} -> {vae.A}")
        if E is not None and int(vae.E) != E:
            raise _lib.PulseError(f"ZTaskStepsB200: the {layout} latent has {E} dimensions (embedding_size), the VAE's {vae.E}")
    if (getattr(policy, "disc", None) is not None) != (amp is not None):
        raise _lib.PulseError("ZTaskStepsB200: a policy with a discriminator needs the AMP part (amp=AmpBuffersB200) and the AMP part a "
                              "discriminator")
    if amp is not None:
        if amp.amp_width != reset.amp_width or amp.upright != reset.upright:
            raise _lib.PulseError(f"ZTaskStepsB200: the AMP part writes {amp.amp_width}-float rows (upright {amp.upright}), the reset "
                                  f"{reset.amp_width}-float rows (upright {reset.upright})")
    return kind


class ZTaskStepsB200(LatentStepsB200):
    """One horizon of a latent-space task per `play_steps()` (the step order, buffers, launch structure and hazards: LatentStepsB200).
    The task's pieces of step t:
         1. reset of the done envs (`ZTaskResetB200.reset_envs`), then the list observation of the reset envs into obses[:, t], then
            `reset_task` (reach, speed);
         5. `pulse_ztask_pre_physics`: PD targets into pd_tar, prev_root_pos (speed, strike), `_update_task` of the due envs (reach, speed);
         7. the rollout step kernel (`pulse_reach_rollout_step` / `pulse_ztask_rollout_step`, SMPL-X: `pulse_smplx_speed_rollout_step` /
            `pulse_smplx_target_rollout_step`).
    `finish()` uses the task reward alone (task_reward_w 1, disc_reward_w 0, pulse_z_task.yaml:90-91).  With the AMP part (`amp`, an
    AmpBuffersB200 of the reset's amp_width and upright setting: 195 floats for env_pulse_amp.yaml) the reset also back-fills the AMP
    history, the driver keeps the horizon's AMP rows and `train_epoch()` trains the discriminator (disc_coef 5) inside the shared
    gradient-norm clip, as pulse_z_task.yaml does (LatentStepsB200); task_reward_w / disc_reward_w then mix the rewards.

    `task`: the ReachTaskB200 / SpeedTaskB200 / StrikeTaskB200 whose targets, change steps and termination settings the steps use.
    `reset`: the ZTaskResetB200 of the same kind.  `policy`: PPOPolicy(obs_size=task.obs_size, num_actions=vae.E, ...).  `vae`: PulseVAE(with_critic=False) holding the frozen prior, decoder and the checkpoint's obs_rms.  `sim`: the
    simulator's tensors, read and written in place through their strides: body_state, root_states, dof_pos, dof_vel, progress_buf,
    sampled_motion_ids, motion_start_times; optional contact_forces, actor_ids, dof_force (the speed task's power term); strike:
    target_states, tar_contact_forces and optional tar_actor_ids.

    The PULSE-X speed task (`HumanoidSpeedZ` with robot=smplx_humanoid) runs through the same driver: `task` a SmplxSpeedTaskB200,
    `reset` a ZTaskResetB200 over a 52-body MotionLib, `policy` PPOPolicy(obs_size=781, num_actions=48), `vae` PulseVAE(self_obs_size=778,
    num_actions=153, latent=48); the sim views hold >= 52 bodies and 153 dofs, and `dof_force` is refused (no power term).

    `policy` may carry a discriminator exactly when `amp` is given (PPOPolicy(..., with_disc=True, amp_obs_size=10 * amp_width)).  For
    the SMPL-X speed task that is AmpBuffersB200(ml, amp_width=465, upright=False, ...) over the same 52-body MotionLib, a reset of
    amp_root_height_obs False and PPOPolicy(obs_size=781, num_actions=48, units=(2048, 1024, 512), act="silu", with_disc=True,
    amp_obs_size=4650).

    The PULSE-X reach and strike tasks take the same pieces with a SmplxReachTaskB200 / SmplxStrikeTaskB200 (obs_size 781 / 793), a
    SmplxTargetResetB200 of the same kind over the 52-body MotionLib, and the same decoder, latent and AMP part.

    The PPO baseline (`HumanoidReach` / `HumanoidSpeed` / `HumanoidStrike` under learning=ppo, the same task trained from scratch):
    `vae=None` and a policy that acts in the dofs, PPOPolicy(obs_size=task.obs_size, num_actions=69 (SMPL) or 153 (SMPL-X),
    units=(2048, 1024, 512), act="silu", logstd=-2.9) (ppo.yaml).  A step is then `heads_into` (critic beside actor on side A),
    `pulse_policy_post` into actions[:, t], neglogp[:, t] and values[t], and `pulse_ztask_pre_physics` on actions[:, t]: no prior,
    latent post-processing or decoder, and no side P.  `actions` and `mus` are [n, T, dofs].  The reset, observations, step kernel,
    next values, AMP part, `finish` and `train_epoch` are those of the latent driver.  The actor head writes its 153-float rows of
    `mus` straight into the strided slice mus[:, t]: the forward epilogue stores fp32 rows with 16-byte stores only when the row
    stride is a multiple of 4 floats and element-wise otherwise, so every horizon T is accepted without padding.

    Out of scope: multi-GPU; Default / Hybrid state init; the power_usage_reward terms the step kernels exclude."""

    def __init__(self, task, reset, policy, vae, sim: dict, horizon: int = 32, pd_offset: Optional[torch.Tensor] = None,
                 pd_scale: Optional[torch.Tensor] = None, pd_freeze: Optional[torch.Tensor] = None, use_graphs: bool = True,
                 gamma: float = 0.99, tau: float = 0.95, reset_seed: int = 0, amp=None, task_reward_w: float = 1.0,
                 disc_reward_w: float = 0.0):
        self.kind = check_pieces(task, reset, policy, vae, amp)
        self.layout = getattr(task, "layout", "smpl")
        missing = [k for k in SIM_KEYS + (STRIKE_KEYS if self.kind == "strike" else ()) if k not in sim]
        if missing:
            raise _lib.PulseError(f"ZTaskStepsB200: sim lacks {missing}")
        if self.layout == "smplx" and sim.get("dof_force") is not None:
            raise _lib.PulseError("ZTaskStepsB200: sim['dof_force'] given, but the SMPL-X steps have no power term")
        n = self.n = int(sim["progress_buf"].shape[0])
        if n != task.num_envs:
            raise _lib.PulseError(f"ZTaskStepsB200: sim has {n} envs, the task {task.num_envs}")
        self._setup(task, reset, policy, vae, sim, horizon, task.obs_size, pd_offset, pd_scale, pd_freeze, use_graphs, gamma, tau, reset_seed,
                    amp, task_reward_w, disc_reward_w)

    # ------------------------------------------------------------------ the pieces of one step
    def _step_args(self, obs: torch.Tensor, rew: torch.Tensor):
        """The task's step arguments with the outputs pointed at experience slices and the driver's reset / terminate words."""
        s, task = self.sim, self.task
        a = task._args(s["body_state"], s["progress_buf"], s.get("contact_forces"))
        if self.kind == "speed":
            task._power_args(a, s.get("dof_force"), s.get("dof_vel"))
        elif self.kind == "strike":
            task._target_args(a, s["target_states"], s["tar_contact_forces"])
        a.obs_buf, a.obs_stride, a.rew_buf = obs.data_ptr(), obs.stride(0), rew.data_ptr()
        a.reset_buf, a.terminate_buf = self.reset_buf.data_ptr(), self.terminate_buf.data_ptr()
        return a

    def _task_kw(self) -> dict:
        task = self.task
        if self.kind == "reach":
            return dict(change_steps=task._tar_change_steps, tar_pos=task._tar_pos)
        return dict(change_steps=task._speed_change_steps, tar_speed=task._tar_speed)

    def _reset(self, t: int) -> None:
        """`env_reset(done_indices)` (amp_agent.py:352) -> HumanoidAMPTask._reset_envs up to the simulator's refresh."""
        s = self.sim
        strike = self.kind == "strike"
        self.reset_ws = self.reset.reset_envs(
            root_states=s["root_states"], dof_pos=s["dof_pos"], dof_vel=s["dof_vel"], rigid_body_state=s["body_state"],
            progress_buf=s["progress_buf"], sampled_motion_ids=s["sampled_motion_ids"], motion_start_times=s["motion_start_times"],
            reset_buf=self.reset_buf, contact_forces=s.get("contact_forces"), amp_obs_buf=self.amp_init if self.amp is not None else None,
            actor_ids=s.get("actor_ids"), target_states=s["target_states"] if strike else None,
            tar_actor_ids=s.get("tar_actor_ids") if strike else None, seed=self.reset_seed, offset=t, offset_dev=self.policy.rng_offset,
            amp_fresh=self.amp_fresh if self.amp is not None else None)

    def _reset_obs(self, t: int) -> None:
        """`_compute_observations(env_ids)` of the reset envs into obses[:, t], then `_reset_task` (humanoid_amp_task.py:66-76)."""
        ws = self.reset_ws
        a = self._step_args(self.obses[:, t], self.rewards[t])
        self._launch(self.task.entries[1], C.byref(a), ws["env_list"].data_ptr(),
                     ws["count"].data_ptr(), self.n)
        if self.kind != "strike":
            self.reset.reset_task(progress_buf=self.sim["progress_buf"], seed=self.reset_seed, offset=t, offset_dev=self.policy.rng_offset,
                                  **self._task_kw())

    def _pre_physics(self, dec: torch.Tensor, t: int, rand: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None) -> None:
        """`pulse_ztask_pre_physics` on the decoder output `dec` [n, dofs] (without a VAE: the sampled actions); `rand` / `steps` inject
        the `_update_task` draws per env."""
        s, task, kind = self.sim, self.task, self.kind
        p = _lib.ZTaskPrePhysicsArgs(kind=task.kind, dofs=self.dofs, action=dec.data_ptr(), ld_action=dec.stride(0), pd_offset=self.pd[0].data_ptr(),
                                     pd_scale=self.pd[1].data_ptr(), freeze=_lib.ptr(self.pd_freeze), pd_out=self.pd_tar.data_ptr(),
                                     ld_pd=self.pd_tar.stride(0), progress_buf=s["progress_buf"].data_ptr(), seed=self.reset_seed, offset=t,
                                     offset_dev=self.policy.rng_offset.data_ptr(), rand=_lib.ptr(rand), steps_in=_lib.ptr(steps))
        if kind != "reach":
            p.root_states, p.root_env_stride, p.prev_root_pos = s["root_states"].data_ptr(), s["root_states"].stride(0), task._prev_root_pos.data_ptr()
        if kind == "reach":
            p.change_steps, p.tar_pos = task._tar_change_steps.data_ptr(), task._tar_pos.data_ptr()
            p.dist_max, p.height_min, p.height_max = task.tar_dist_max, task.tar_height_min, task.tar_height_max
            p.steps_min, p.steps_max = task.tar_change_steps_min, task.tar_change_steps_max
        elif kind == "speed":
            p.change_steps, p.tar_speed = task._speed_change_steps.data_ptr(), task._tar_speed.data_ptr()
            p.speed_scale, p.speed_min = task._tar_speed_max - task._tar_speed_min, task._tar_speed_min
            p.steps_min, p.steps_max = task._speed_change_steps_min, task._speed_change_steps_max
        self._launch("pulse_ztask_pre_physics", C.byref(p), self.n)

    def _env_step(self, t: int) -> None:
        """post_physics_step (humanoid.py:1315-1346): one fused launch."""
        a = self._step_args(self._next_obs(t), self.rewards[t])
        self._launch(self.task.entries[2], C.byref(a), self.dones[t].data_ptr(), self.n)

    def first_observation(self) -> None:
        """Observation of the initial state (Humanoid.reset -> _compute_observations at start-up): fills `obs_carry`."""
        a = self._step_args(self.obs_carry, self.rewards[0])
        self._launch(self.task.entries[0], C.byref(a), self.n)
        self.reset_buf.zero_()
        self.terminate_buf.zero_()
        self._amp_start()
