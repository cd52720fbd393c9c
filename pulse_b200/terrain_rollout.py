"""The pedestrian terrain task's training iteration on the device: the rollout of HumanoidPedestrianTerrainZ (pulse_z_terrain.yaml with
env_pulse_terrain.yaml) with the `amp_sept` latent policy, the frozen PULSE prior + decoder and the device reset, then GAE and the PPO
update (`AMPAgent.play_steps` + `train_epoch`, phc/learning/amp_agent.py:341-439; `HumanoidAMPTask` resets, humanoid_amp_task.py:57-76;
`HumanoidZ.step -> step_z`, humanoid_z.py:157-173)."""
import ctypes as C
from typing import List, Optional, Tuple

import torch

from . import _lib
from .latent_rollout import LatentStepsB200
from .sept import SeptPolicy
from .terrain import SELF_OBS, PedestrianTerrainTaskB200
from .terrain_reset import TerrainResetB200
from .vae import pd_targets

SIM_KEYS = ("body_state", "root_states", "dof_pos", "dof_vel", "progress_buf", "sampled_motion_ids", "motion_start_times")


def _same_heightfield(a, b) -> bool:
    """Whether two TerrainB200 sample the same heightfield: the same sizes, scales and cells.  The task and the reset usually hold
    separate uploads of one map (each `from_reference` call uploads its own copy), so the cells are compared, once, at construction."""
    if a is b:
        return True
    if a.heightfield is None or b.heightfield is None:
        return False
    if (a.rows, a.cols, a.horizontal_scale, a.vertical_scale) != (b.rows, b.cols, b.horizontal_scale, b.vertical_scale):
        return False
    return a.heightfield.data_ptr() == b.heightfield.data_ptr() or torch.equal(a.heightfield, b.heightfield.to(a.heightfield.device))


def check_pieces(task, reset, policy, vae, amp=None) -> None:
    """Checks that the step object, the reset, the sept policy and the frozen VAE belong together; raises PulseError naming the mismatch."""
    who = "TerrainStepsB200"
    if not isinstance(task, PedestrianTerrainTaskB200):
        raise _lib.PulseError(f"{who}: task must be a PedestrianTerrainTaskB200")
    if task.terrain.heightfield is None:
        raise _lib.PulseError(f"{who}: plane terrain: the reset cannot spawn on a plane (the reference builds no walkable table for it)")
    if not isinstance(reset, TerrainResetB200):
        raise _lib.PulseError(f"{who}: reset must be a TerrainResetB200")
    if not _same_heightfield(reset.terrain, task.terrain):
        raise _lib.PulseError(f"{who}: the reset and the task sample different heightfields")
    if not isinstance(policy, SeptPolicy):
        raise _lib.PulseError(f"{who}: policy must be a SeptPolicy (the amp_sept network of pulse_z_terrain.yaml)")
    if (getattr(policy, "disc", None) is not None) != (amp is not None):
        raise _lib.PulseError(f"{who}: a policy with a discriminator needs the AMP part (amp=AmpBuffersB200) and the AMP part a discriminator")
    if amp is not None and (amp.amp_width != reset.amp_width or amp.upright != reset.upright):
        raise _lib.PulseError(f"{who}: the AMP part writes {amp.amp_width}-float rows (upright {amp.upright}), the reset {reset.amp_width}-float "
                              f"rows (upright {reset.upright})")
    W = int(task.get_obs_size())
    if int(policy.S) + int(policy.task_in) != W:
        raise _lib.PulseError(f"{who}: the task writes {W} observation floats, the policy reads {policy.S} + {policy.task_in}")
    if int(policy.S) != SELF_OBS or int(vae.S) != SELF_OBS:
        raise _lib.PulseError(f"{who}: the self observation has {SELF_OBS} floats, the policy reads {policy.S} and the VAE {vae.S}")
    if int(policy.A) != int(vae.E):
        raise _lib.PulseError(f"{who}: the policy acts in {policy.A} dimensions, the VAE's latent has {vae.E}")
    if int(vae.A) != 69:
        raise _lib.PulseError(f"{who}: the decoder must produce 69 dof targets, not {vae.A}")


def philox_blocks(env: int, t: int, rng_offset: int, latent: int = 32) -> List[Tuple[str, int, int]]:
    """The Philox4x32-10 blocks step t of a horizon reads for `env`, as (key, index, counter), with `rng_offset` the policy's device
    offset at the start of the horizon (it moves on by the horizon length after each one).  key 'reset' is the driver's reset seed,
    'policy' the policy's sampling seed (include/pulse_b200.h):
        pulse_reset_terrain      index env, counter rng_offset + t (clip, start time, spawn location);
        pulse_traj_reset_list    index env + 4 * 2^32, counters PULSE_TRAJ_VERTS * (rng_offset + t) + k, k < PULSE_TRAJ_VERTS;
        pulse_latent_post        index env * 64 + p for the latent pairs p < ceil(latent / 2), counter rng_offset + t."""
    off = rng_offset + t
    index, counters = _lib.traj_list_philox_blocks(env, t, rng_offset)
    return ([("reset", env, off)] + [("reset", index, c) for c in counters]
            + [("policy", env * 64 + p, off) for p in range((latent + 1) // 2)])


class TerrainStepsB200(LatentStepsB200):
    """One horizon of HumanoidPedestrianTerrainZ per `play_steps()` (the step order, buffers, launch structure and hazards:
    LatentStepsB200).  For every step t, in the reference's order (amp_agent.py:341-439, humanoid_z.py:157-173,
    humanoid_amp_task.py:57-76):
         1. reset of the done envs: `TerrainResetB200.reset_envs` (no AMP buffer, Philox clip / start-time / location draws keyed
            (reset_seed, env, t + the policy's device offset)), then the `refresh(t, ws)` hook if set;
         2. the list observation of the reset envs into obses[:, t] (`pulse_terrain_step`, PULSE_STEP_OBS over the reset's env list and
            count); it still samples the previous episode's waypoints, as the reference does;
         3. new waypoints of the reset envs (`TerrainResetB200.reset_task`, `pulse_traj_reset_list`);
         4. `heads_into`: the normalise split and the task encoder once, then the actor beside the critic; beside them, on side P, the
            frozen prior on obses[:, t, :358];
         5. `pulse_latent_post`, the decoder, then `pulse_pd_targets` into pd_tar (the terrain task has no `_update_task` and no
            prev_root_pos);
         6. the caller's `physics(t)` hook;
         7. `pulse_terrain_rollout_step` (progress += 1, reward, reset, next observation) into obses[:, t+1] / obs_carry, rewards[t],
            dones[t], reset_buf and terminate_buf;
         8. next_values[t] = critic(obses[:, t+1]) (1 - terminate) on slot 1, on side B.
    `finish()` uses the task reward alone (task_reward_w 1, disc_reward_w 0) and `train_epoch()` runs `SeptPolicy.train_minibatch` over
    contiguous row ranges with old_mu = mus.  The Philox blocks a step reads: `philox_blocks`.

    Hazard beside those of LatentStepsB200: side B's next values run the task encoder too.  They normalise into the slot-1 operands
    (x_next, t_next) and run the encoder and the critic on their slot-1 workspaces; `heads_into` on main uses the slot-0 operands
    (x, t) and workspaces, so the encoder of step t+1 on main and the one of step t on B share no buffer.

    `task`: a PedestrianTerrainTaskB200 on a heightfield; its traj_verts are the waypoints the steps read and the resets rewrite, and the
    caller provides the initial ones (e.g. `task.reset_task` over all envs) before `first_observation()`.  `reset`: the
    TerrainResetB200 over the same heightfield (same sizes, scales and cells, compared once at construction: the task and the reset
    may hold separate uploads of the map, as two `from_reference` calls make them).  `policy`: SeptPolicy(num_actions=vae.E, ...) whose self + task
    observation is the task's (358 + 1044 = 1402 floats for env_pulse_terrain.yaml).  `vae`: PulseVAE(with_critic=False) holding the
    frozen prior, decoder and the checkpoint's obs_rms.  `sim`: the simulator's tensors, read and written in place through their
    strides: body_state, root_states, dof_pos, dof_vel, progress_buf, sampled_motion_ids, motion_start_times (the terrain reset's
    clip / start-time buffers); contact_forces with early termination; dof_force with power_reward; optional actor_ids.

    With the AMP part (`amp`, an AmpBuffersB200 of the reset's layout, 196 floats for env_pulse_terrain.yaml, given exactly when the
    policy has a discriminator) the reset back-fills the AMP history and `train_epoch()` trains the discriminator inside the shared
    gradient-norm clip, as pulse_z_terrain.yaml does (LatentStepsB200).

    Out of scope: multi-GPU; group observations and the velocity map; mesh terrain; Default / Hybrid state init; an agent
    mixin (INTEGRATION.md wires the hooks)."""

    def __init__(self, task, reset, policy, vae, sim: dict, horizon: int = 32, pd_offset: Optional[torch.Tensor] = None,
                 pd_scale: Optional[torch.Tensor] = None, pd_freeze: Optional[torch.Tensor] = None, use_graphs: bool = True,
                 gamma: float = 0.99, tau: float = 0.95, reset_seed: int = 0, amp=None, task_reward_w: float = 1.0,
                 disc_reward_w: float = 0.0):
        check_pieces(task, reset, policy, vae, amp)
        keys = SIM_KEYS + (("contact_forces",) if task.enable_early_termination else ()) + (("dof_force",) if task.power_reward else ())
        missing = [k for k in keys if sim.get(k) is None]
        if missing:
            raise _lib.PulseError(f"TerrainStepsB200: sim lacks {missing}")
        n = self.n = int(sim["progress_buf"].shape[0])
        if n != task.num_envs:
            raise _lib.PulseError(f"TerrainStepsB200: sim has {n} envs, the task {task.num_envs}")
        self._setup(task, reset, policy, vae, sim, horizon, task.get_obs_size(), pd_offset, pd_scale, pd_freeze, use_graphs, gamma, tau,
                    reset_seed, amp, task_reward_w, disc_reward_w)

    # ------------------------------------------------------------------ the task's pieces of one step
    def _step_args(self, flags: int, obs: torch.Tensor, rew: torch.Tensor):
        """The task's step arguments with the outputs pointed at experience slices and the driver's reset / terminate words."""
        s, task = self.sim, self.task
        a = task._step_args(flags, s["body_state"], s["root_states"], s["progress_buf"])
        if task.enable_early_termination:
            a.contact_forces, a.contact_env_stride = s["contact_forces"].data_ptr(), s["contact_forces"].stride(0)
        if task.power_reward:
            a.dof_force, a.dof_force_stride = s["dof_force"].data_ptr(), s["dof_force"].stride(0)
            a.dof_vel, a.dof_env_stride, a.dof_elem_stride = s["dof_vel"].data_ptr(), s["dof_vel"].stride(0), s["dof_vel"].stride(1)
        a.obs_buf, a.obs_stride, a.rew_buf = obs.data_ptr(), obs.stride(0), rew.data_ptr()
        a.reset_buf, a.terminate_buf = self.reset_buf.data_ptr(), self.terminate_buf.data_ptr()
        return a

    def _reset(self, t: int) -> None:
        """`env_reset(done_indices)` (amp_agent.py:352) -> HumanoidAMPTask._reset_envs up to the simulator's refresh."""
        s = self.sim
        self.reset_ws = self.reset.reset_envs(
            root_states=s["root_states"], dof_pos=s["dof_pos"], dof_vel=s["dof_vel"], rigid_body_state=s["body_state"],
            progress_buf=s["progress_buf"], sampled_motion_ids=s["sampled_motion_ids"], motion_start_times=s["motion_start_times"],
            reset_buf=self.reset_buf, contact_forces=s.get("contact_forces"), amp_obs_buf=self.amp_init if self.amp is not None else None,
            actor_ids=s.get("actor_ids"), seed=self.reset_seed, offset=t, offset_dev=self.policy.rng_offset,
            amp_fresh=self.amp_fresh if self.amp is not None else None)

    def _reset_obs(self, t: int) -> None:
        """`_compute_observations(env_ids)` of the reset envs into obses[:, t], then `_reset_task` (humanoid_amp_task.py:66-76)."""
        ws = self.reset_ws
        a = self._step_args(_lib.STEP_OBS, self.obses[:, t], self.rewards[t])
        a.env_ids, a.env_count = ws["env_list"].data_ptr(), ws["count"].data_ptr()
        self._launch("pulse_terrain_step", C.byref(a), self.n)
        self.reset.reset_task(self.task, self.sim["root_states"], seed=self.reset_seed, offset=t, offset_dev=self.policy.rng_offset)

    def _pre_physics(self, dec: torch.Tensor, t: int) -> None:
        """pre_physics_step: the PD targets of the decoder output (humanoid.py:1222-1247, `pulse_pd_targets`)."""
        pd_targets(dec, self.pd[0], self.pd[1], out=self.pd_tar, freeze=self.pd_freeze)

    def _env_step(self, t: int) -> None:
        """post_physics_step (humanoid.py:1315-1346): one fused launch."""
        a = self._step_args(_lib.STEP_ALL, self._next_obs(t), self.rewards[t])
        self._launch("pulse_terrain_rollout_step", C.byref(a), self.dones[t].data_ptr(), self.n)

    def first_observation(self) -> None:
        """Observation of the initial state (Humanoid.reset -> _compute_observations at start-up) into `obs_carry`, from the waypoints
        the caller has put into task.traj_verts."""
        a = self._step_args(_lib.STEP_OBS, self.obs_carry, self.rewards[0])
        self._launch("pulse_terrain_step", C.byref(a), self.n)
        self.reset_buf.zero_()
        self.terminate_buf.zero_()
        self._amp_start()
