"""The VR controller task's training iteration on the device: the rollout of HumanoidImZ (pulse_z_vr.yaml with env_pulse_im.yaml:
the latent policy tracks the head and both hands through the frozen PULSE prior + decoder) with the device reset, then GAE and the PPO
update (`AMPAgent.play_steps` + `train_epoch`, phc/learning/amp_agent.py:341-439; `Humanoid.reset -> _reset_envs`, humanoid.py:526-587;
`HumanoidZ.step -> step_z`, humanoid_z.py:157-173)."""
from typing import List, Optional, Tuple

import torch

from . import _lib
from .humanoid_im import SELF_OBS, HumanoidImCompute
from .latent_rollout import LatentStepsB200
from .vae import pd_targets

SIM_KEYS = ("body_state", "root_states", "dof_pos", "dof_vel", "progress_buf", "motion_ids", "motion_start_times", "motion_start_offset",
            "global_offset")


def compute_from_task(task) -> HumanoidImCompute:
    """The `HumanoidImCompute` of a live HumanoidImZ task: the settings `HumanoidImB200Mixin` reads, plus its tracked bodies
    (`_track_bodies_id`, in the task's order) and observation version (`obs_v`; 4 and 6 share a function, humanoid_im.py:786-787).
    Refuses, naming them, the task settings under which the task's observation is not the tracked row."""
    obs_v = int(getattr(task, "obs_v", 6))
    obs_v = 6 if obs_v == 4 else obs_v
    unsupported = [name for name, bad in (
        ("obs_v %d (the tracked row serves 4, 6 and 7)" % obs_v, obs_v not in (6, 7)),
        ("fut_tracks", bool(getattr(task, "_fut_tracks", False))),
        ("zero_out_far", bool(getattr(task, "zero_out_far", False))),
        ("occlusion", bool(getattr(task, "_occl_training", False))),
        ("full_body_reward False", not bool(getattr(task, "_full_body_reward", True))),
        ("self_obs_v %s" % getattr(task, "self_obs_v", 1), int(getattr(task, "self_obs_v", 1)) != 1),
        ("observation noise", bool(getattr(task, "add_obs_noise", False))),
        ("a non-upright start", not bool(getattr(task, "_has_upright_start", True)))) if bad]
    if unsupported:
        raise _lib.PulseError(f"compute_from_task: the tracked row does not serve {', '.join(unsupported)}")
    return HumanoidImCompute.from_task(task, track_body_ids=tuple(int(j) for j in task._track_bodies_id), obs_version=obs_v)


def check_pieces(comp, policy, vae, amp=None) -> None:
    """Checks that the tracked-body compute, the latent policy and the frozen VAE belong together; raises PulseError naming the mismatch."""
    who = "ImZStepsB200"
    if not isinstance(comp, HumanoidImCompute) or comp.track is None:
        raise _lib.PulseError(f"{who}: comp must be a HumanoidImCompute with a tracked configuration (ImConfig.track_body_ids)")
    if comp.cfg.cycle_motion:
        raise _lib.PulseError(f"{who}: cycle_motion is not supported (its start-time rewrite of wrapped envs runs on the host)")
    if comp.cfg.use_mean_reset:
        raise _lib.PulseError(f"{who}: use_mean_reset (the im_eval criterion) is an evaluation setting, not a training one")
    if (getattr(policy, "disc", None) is not None) != (amp is not None):
        raise _lib.PulseError(f"{who}: a policy with a discriminator needs the AMP part (amp=AmpBuffersB200) and the AMP part a discriminator")
    if amp is not None and (amp.amp_width != 196 or not amp.upright):
        raise _lib.PulseError(f"{who}: the reference-state reset back-fills 196-float upright AMP rows, the AMP part has {amp.amp_width} "
                              f"(upright {amp.upright})")
    if int(policy.obs_size) != comp.obs_size:
        raise _lib.PulseError(f"{who}: the tracked observation has {comp.obs_size} floats, the policy reads {policy.obs_size}")
    if int(vae.S) != SELF_OBS or int(vae.A) != 69:
        raise _lib.PulseError(f"{who}: the decoder must map the {SELF_OBS}-float self observation to 69 dof targets, not {vae.S} -> {vae.A}")
    if int(policy.A) != int(vae.E):
        raise _lib.PulseError(f"{who}: the policy acts in {policy.A} dimensions, the VAE's latent has {vae.E}")


def philox_blocks(env: int, t: int, rng_offset: int, latent: int = 32) -> List[Tuple[str, int, int]]:
    """The Philox4x32-10 blocks step t of a horizon reads for `env`, as (key, index, counter), with `rng_offset` the policy's device
    offset at the start of the horizon (it moves on by the horizon length after each one).  key 'reset' is the driver's reset seed,
    'policy' the policy's sampling seed (include/pulse_b200.h):
        pulse_reset_ref_state    index env, counter rng_offset + t (the start-time draw, word 0);
        pulse_latent_post        index env * 64 + p for the latent pairs p < ceil(latent / 2), counter rng_offset + t."""
    off = rng_offset + t
    return [("reset", env, off)] + [("policy", env * 64 + p, off) for p in range((latent + 1) // 2)]


class ImZStepsB200(LatentStepsB200):
    """One horizon of HumanoidImZ per `play_steps()` (the step order, buffers, launch structure and hazards: LatentStepsB200).  For every
    step t, in the reference's order (amp_agent.py:341-439, humanoid.py:526-587, humanoid_z.py:157-173):
         1. reset of the done envs: `HumanoidImCompute.reset_envs` in mask mode (`pulse_reset_ref_state`: reference-state episodes, no
            AMP buffer, the Philox start-time draw keyed (reset_seed, env, t + the policy's device offset)), then the `refresh(t, ws)`
            hook if set;
         2. the observation of the reset envs into obses[:, t]: `pulse_im_track_step` with PULSE_STEP_OBS over the reset's env list and
            device-side count (HumanoidIm's `_reset_task` does nothing);
         3. `heads_into`: the actor beside the critic; beside them, on side P, the frozen prior on obses[:, t, :358];
         4. `pulse_latent_post`, the decoder, then `pulse_pd_targets` into pd_tar (`_update_cycle_count` does nothing without
            cycle_motion);
         5. the caller's `physics(t)` hook;
         6. `pulse_im_track_step` with PULSE_STEP_ALL | PULSE_STEP_ADVANCE (progress += 1, full-body reward and reset, the tracked
            next observation) into obses[:, t+1] / obs_carry, rewards[t], dones[t], reset_buf and terminate_buf;
         7. next_values[t] = critic(obses[:, t+1]) (1 - terminate) on slot 1, on side B.
    `finish()` uses the task reward alone (task_reward_w 1, disc_reward_w 0) and `train_epoch()` runs `PPOPolicy.train_minibatch` over
    contiguous row ranges with old_mu = mus.  The Philox blocks a step reads: `philox_blocks`.

    `comp`: a HumanoidImCompute with `track_body_ids` set (`compute_from_task(task)` builds it from a live task with the settings the
    HumanoidIm mixin reads); its MotionLib serves the reset and the steps.  `policy`: PPOPolicy(obs_size=comp.obs_size,
    num_actions=vae.E, units=(2048, 1536, 1024, 1024, 512, 512), act="silu", logstd=-1.5) (pulse_z_vr.yaml).
    `vae`: PulseVAE(with_critic=False) holding the frozen prior, decoder and the checkpoint's obs_rms.  `sim`: the simulator's and the
    task's tensors, read and written in place through their strides: body_state, root_states, dof_pos, dof_vel, progress_buf,
    motion_ids (`_sampled_motion_ids`), motion_start_times, motion_start_offset (`_motion_start_times_offset`), global_offset;
    dof_force with power_reward; optional contact_forces (cleared for the reset envs) and actor_ids.

    With the AMP part (`amp`, an AmpBuffersB200 of 196-float upright rows over the comp's MotionLib, given exactly when the policy has a
    discriminator) the reset back-fills the AMP history through pulse_reset_ref_state's AMP path and `train_epoch()` trains the
    discriminator inside the shared gradient-norm clip, as pulse_z_vr.yaml does (LatentStepsB200).

    Out of scope: the fut_tracks windows, observation versions 1/2/3/8/9, non-upright starts, zero_out_far and occlusion;
    multi-GPU; the smplx humanoid; an agent mixin (INTEGRATION.md wires the hooks).  The IMAmpAgent evaluation pass is `evaluate`."""

    def __init__(self, comp: HumanoidImCompute, policy, vae, sim: dict, horizon: int = 32, pd_offset: Optional[torch.Tensor] = None,
                 pd_scale: Optional[torch.Tensor] = None, pd_freeze: Optional[torch.Tensor] = None, use_graphs: bool = True,
                 gamma: float = 0.99, tau: float = 0.95, reset_seed: int = 0, amp=None, task_reward_w: float = 1.0,
                 disc_reward_w: float = 0.0):
        check_pieces(comp, policy, vae, amp)
        keys = SIM_KEYS + (("dof_force",) if comp.cfg.power_reward else ())
        missing = [k for k in keys if sim.get(k) is None]
        if missing:
            raise _lib.PulseError(f"ImZStepsB200: sim lacks {missing}")
        self.n = int(sim["progress_buf"].shape[0])
        self.comp = comp
        self._setup(comp, comp, policy, vae, sim, horizon, comp.obs_size, pd_offset, pd_scale, pd_freeze, use_graphs, gamma, tau, reset_seed,
                    amp, task_reward_w, disc_reward_w)

    # ------------------------------------------------------------------ the task's pieces of one step
    def _state(self) -> dict:
        s = self.sim
        return dict(body_state=s["body_state"], progress_buf=s["progress_buf"], motion_ids=s["motion_ids"],
                    motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"])

    def _reset(self, t: int) -> None:
        """`env_reset(done_indices)` (amp_agent.py:352) -> Humanoid._reset_envs up to the simulator's refresh."""
        s = self.sim
        self.reset_ws = self.comp.reset_envs(
            motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
            global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
            dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=self.reset_buf, contact_forces=s.get("contact_forces"),
            actor_ids=s.get("actor_ids"), seed=self.reset_seed, offset=t, offset_dev=self.policy.rng_offset,
            amp_obs_buf=self.amp_init if self.amp is not None else None, amp_fresh=self.amp_fresh if self.amp is not None else None)

    def _reset_obs(self, t: int) -> None:
        """`_compute_observations(env_ids)` of the reset envs into obses[:, t] (HumanoidIm's `_reset_task` does nothing)."""
        ws = self.reset_ws
        self.comp.step(flags=_lib.STEP_OBS, obs_buf=self.obses[:, t], env_ids=ws["env_list"], env_count=ws["count"], **self._state())

    def _pre_physics(self, dec: torch.Tensor, t: int) -> None:
        """pre_physics_step: the PD targets of the decoder output (humanoid.py:1222-1247, `pulse_pd_targets`)."""
        pd_targets(dec, self.pd[0], self.pd[1], out=self.pd_tar, freeze=self.pd_freeze)

    def _env_step(self, t: int) -> None:
        """post_physics_step (humanoid.py:1315-1346): one fused launch."""
        s = self.sim
        self.comp.step(flags=_lib.STEP_ALL, advance=True, obs_buf=self._next_obs(t), rew_buf=self.rewards[t], reset_buf=self.reset_buf,
                       terminate_buf=self.terminate_buf, fdones_out=self.dones[t], dof_force=s.get("dof_force"), dof_vel=s["dof_vel"],
                       **self._state())

    def first_observation(self) -> None:
        """Observation of the initial state (Humanoid.reset -> _compute_observations at start-up) into `obs_carry`."""
        self.comp.step(flags=_lib.STEP_OBS, obs_buf=self.obs_carry, **self._state())
        self.reset_buf.zero_()
        self.terminate_buf.zero_()
        self._amp_start()

    def evaluate(self, dataset, physics=None, auto_pmcp: bool = False, auto_pmcp_soft: bool = False, **kw):
        """`IMAmpAgent.eval` (im_amp.py:136-242) of this policy over every clip of `dataset` (a MotionDatasetB200) on this driver's
        simulator tensors, then every env reset into training and the optional PMCP update: `evaluation.EvalStepsB200` (`kw`: its
        poll_every / use_graphs / strict_eval / eval_body_ids).  The pass is `self.eval_steps` while it runs: `physics(t)` applies
        its `pd_tar` and may read its task-side state (`progress_buf`, `motion_start_times`, ...)."""
        from .evaluation import EvalStepsB200
        self.eval_steps = EvalStepsB200(self, physics=physics, **kw)
        return self.eval_steps.run(dataset, auto_pmcp=auto_pmcp, auto_pmcp_soft=auto_pmcp_soft)
