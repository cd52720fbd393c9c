"""PULSE's distillation iteration on the device: the rollout of HumanoidImDistillGetup with the frozen teacher and the VAE student,
and the only_kin_loss update (`AMPAgent.play_steps` + `_optimize_kin` with only_kin_loss: True, phc/learning/amp_agent.py:341-439,
:771-849; env_im_vae.yaml + im_z_fit.yaml)."""
import ctypes as C
from typing import Callable, Optional

import torch

from . import _lib
from .rollout import GraphRunner

GETUP_KEYS = ("recovery_counter", "available_fall_states", "fall_id_assignments", "fall_root_states", "fall_dof_pos", "fall_dof_vel",
              "recovery_prob", "fall_prob", "recovery_steps")


class DistillStepsB200(GraphRunner):
    """One horizon of the distillation rollout per `play_steps()`, for every step t:
         1. getup reset of the done envs (`reset_getup`, Philox draws keyed (seed, env, t + the student's device offset)), the
            `refresh(t, ws)` hook if set, the observation of the reset envs into obses[:, t];
         2. the teacher (`TeacherPNN`) on obses[:, t] into kin_gt[:, t]  (HumanoidImDistill.step, humanoid_im_distill.py:152-205);
         3. the student (`PulseVAE.act_into`: eval-mode encoder, in-kernel reparameterisation, decoder) into mus[:, t];
         4. `pulse_distill_pre_physics`: PD targets from mus[:, t], kin_progress[:, t] = progress_buf, recovery_counter decremented;
         5. the caller's `physics(t)` hook;
         6. the fused step kernel (progress += 1, reward, reset, next observation, recovery masking) into obses[:, t+1] / obs_carry,
            rewards[t], dones[t], reset_buf, terminate_buf.
    The experience buffers are env-major (`obses[n, T, 934]`, `kin_gt[n, T, A]`, `kin_progress[n, T]`, `mus[n, T, A]`): an update
    minibatch is a contiguous row range of the flattened buffers, the layout `PulseVAE.optimize_kin` takes.

    Not computed (only_kin_loss: none of it reaches `_optimize_kin` or the weights a distilled checkpoint is loaded from): critic values
    and next values, AMP observations and their history, discriminator rewards, GAE / returns, the value / AMP statistics merges, the AMP
    replay buffer.  The checkpoint's value and AMP statistics therefore stay as loaded, and `rewards` holds the task reward only.

    `sim`: the simulator's tensors as `PlayStepsB200` takes them.  `getup`: the task's recovery_counter (int32 [n]), available_fall_states,
    fall_id_assignments, fall_root_states / fall_dof_pos / fall_dof_vel (the fall pool), recovery_prob, fall_prob, recovery_steps; the
    tensors are updated in place.
    Launch structure: with no hooks the whole horizon is ONE CUDA graph, the teacher of step t on a side stream beside the student, the
    pre-physics kernel, the step kernel and the reset of step t+1; with hooks the steps run as graph segments between the hook calls."""

    def __init__(self, comp, vae, teacher, sim: dict, getup: dict, horizon: int = 32, pd_offset: Optional[torch.Tensor] = None,
                 pd_scale: Optional[torch.Tensor] = None, pd_freeze: Optional[torch.Tensor] = None, use_graphs: bool = True, reset_seed: int = 0):
        missing = [k for k in GETUP_KEYS if k not in getup]
        if missing:
            raise _lib.PulseError(f"DistillStepsB200: getup lacks {missing}")
        if int(vae.horizon) != int(horizon):
            raise _lib.PulseError(f"DistillStepsB200: the student's AR(1) horizon {vae.horizon} differs from the rollout horizon {horizon}")
        if teacher.A != vae.A or teacher.obs_size != vae.obs_size:
            raise _lib.PulseError("DistillStepsB200: teacher and student must share the observation and action sizes")
        self.comp, self.vae, self.teacher, self.sim, self.getup, self.T = comp, vae, teacher, sim, getup, int(horizon)
        self.dev = comp.device
        self.lib = _lib.load()
        n = self.n = int(sim["progress_buf"].shape[0])
        T, A, dev = self.T, vae.A, self.dev
        rc = getup["recovery_counter"]
        if rc.dtype != torch.int32 or not rc.is_contiguous() or rc.shape[0] != n:
            raise _lib.PulseError("getup['recovery_counter'] must be contiguous int32 [n]")
        z = lambda *s, **k: torch.zeros(*s, device=dev, **k)
        self.obses, self.obs_carry = z(n, T, vae.obs_size), z(n, vae.obs_size)
        self.kin_gt, self.mus = z(n, T, A), z(n, T, A)
        self.kin_progress = z(n, T, dtype=torch.int64)
        self.rewards, self.dones = z(T, n), z(T, n)
        self.reward_raw = z(n, 5)
        self.reset_buf, self.terminate_buf = z(n, dtype=torch.long), z(n, dtype=torch.long)
        self.pd_tar = z(n, A)
        self.pd = (pd_offset if pd_offset is not None else z(A), pd_scale if pd_scale is not None else torch.ones(A, device=dev))
        if pd_freeze is not None and (pd_freeze.dtype != torch.uint8 or pd_freeze.numel() != A):
            raise _lib.PulseError(f"pd_freeze must be uint8 [{A}]")
        self.pd_freeze = pd_freeze
        self.reset_seed = (int(reset_seed) * 0x9E3779B97F4A7C15 + 0x13198A2E03707344) & (2 ** 64 - 1)
        self.use_graphs = use_graphs
        self._graphs, self._pool = {}, None
        self.physics: Optional[Callable[[int], None]] = None           # physics(t): between the pre-physics kernel and the step kernel
        self.refresh: Optional[Callable[[int, dict], None]] = None     # refresh(t, ws): after the reset, before the reset envs' observation
        self.teacher_side = True            # False: the teacher runs on the main stream (the measurement's comparison schedule)
        self.reset_ws = None
        self._side = None
        self._kld = None
        self.mb_stats = None

    # ------------------------------------------------------------------ the pieces of one step
    def _step_kw(self):
        s = self.sim
        return dict(body_state=s["body_state"], dof_vel=s["dof_vel"], dof_force=s["dof_force"], progress_buf=s["progress_buf"],
                    motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                    global_offset=s["global_offset"], cycle_counter=s.get("cycle_counter"), reward_raw=self.reward_raw,
                    reset_buf=self.reset_buf, terminate_buf=self.terminate_buf)

    def _reset(self, t: int) -> None:
        """`env_reset(done_indices)` (amp_agent.py:352) -> HumanoidImGetup._reset_envs / _reset_actors (humanoid_im_getup.py:135-188)."""
        s, g = self.sim, self.getup
        self.reset_ws = self.comp.reset_getup(
            motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
            global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
            dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=self.reset_buf, terminate_buf=self.terminate_buf,
            recovery_counter=g["recovery_counter"], available_fall_states=g["available_fall_states"],
            fall_id_assignments=g["fall_id_assignments"], fall_root_states=g["fall_root_states"], fall_dof_pos=g["fall_dof_pos"],
            fall_dof_vel=g["fall_dof_vel"], recovery_prob=g["recovery_prob"], fall_prob=g["fall_prob"], recovery_steps=g["recovery_steps"],
            cycle_counter=s.get("cycle_counter"), contact_forces=s.get("contact_forces"), actor_ids=s.get("actor_ids"),
            seed=self.reset_seed, offset=t, offset_dev=self.vae.rng_offset)

    def _reset_obs(self, t: int) -> None:
        """`_compute_observations(env_ids)` of the reset envs, on the device-side list the reset left."""
        s, ws = self.sim, self.reset_ws
        self.comp.step(body_state=s["body_state"], progress_buf=s["progress_buf"], motion_ids=s["motion_ids"],
                       motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"],
                       obs_buf=self.obses[:, t], env_ids=ws["env_list"][:self.n], env_count=ws["count"], flags=_lib.STEP_OBS)

    def _teacher(self, t: int, side) -> None:
        """The teacher of step t, on `side` when given: it waits for obses[:, t] to be final and is joined later by the caller."""
        if side is None:
            self.teacher.gt_action(self.obses[:, t], out=self.kin_gt[:, t])
            return
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        side.wait_event(ev)
        with torch.cuda.stream(side):
            self.teacher.gt_action(self.obses[:, t], out=self.kin_gt[:, t])

    def _act(self, t: int) -> None:
        """The student's action (amp_agent.py:359-369 in eval mode) and the pre-physics launch (PD targets, progress record,
        `_update_recovery_count`, humanoid_im_getup.py:76-80)."""
        self.vae.act_into(self.obses[:, t], mus=self.mus[:, t], rng_step=t)
        mus, kp, rc = self.mus[:, t], self.kin_progress[:, t], self.getup["recovery_counter"]
        with torch.cuda.device(self.dev):
            _lib.check(self.lib.pulse_distill_pre_physics(mus.data_ptr(), mus.stride(0), self.pd[0].data_ptr(), self.pd[1].data_ptr(),
                                                          _lib.ptr(self.pd_freeze), self.n, self.vae.A, self.pd_tar.data_ptr(), self.pd_tar.stride(0),
                                                          self.sim["progress_buf"].data_ptr(), kp.data_ptr(), kp.stride(0), rc.data_ptr(),
                                                          _lib.current_stream(self.dev)), "pulse_distill_pre_physics")

    def _env_step(self, t: int) -> None:
        """post_physics_step (humanoid.py:1315-1346, humanoid_im_getup.py:203-210): one fused launch."""
        nxt = self.obses[:, t + 1] if t + 1 < self.T else self.obs_carry
        self.comp.step(obs_buf=nxt, rew_buf=self.rewards[t], fdones_out=self.dones[t], advance=True,
                       recovery_counter=self.getup["recovery_counter"], **self._step_kw())

    def _side_stream(self):
        if not self.teacher_side:
            return None
        if self._side is None:
            self._side = torch.cuda.Stream(self.dev)
        return self._side

    # ------------------------------------------------------------------ schedules
    def _whole(self) -> None:
        """The horizon as one launch sequence.  The teacher of step t waits only for the event after obses[:, t] is final and runs beside
        the student, the pre-physics kernel, the step kernel and the reset of step t+1; nothing on the main stream writes what it reads
        (obses[:, t] is written before the event and never again in the horizon, the teacher's operand and workspaces are its own), and
        consecutive teacher chains are ordered by their stream.  The main stream joins the side stream once, at the end."""
        side = self._side_stream()
        for t in range(self.T):
            self._reset(t)
            self._reset_obs(t)
            self._teacher(t, side)
            self._act(t)
            self._env_step(t)
        if side is not None:
            torch.cuda.current_stream(self.dev).wait_stream(side)

    def _act_segment(self, t: int) -> None:
        """Segment mode: the observation of the reset envs, then teacher beside student + pre-physics, joined inside the segment."""
        side = self._side_stream()
        self._reset_obs(t)
        self._teacher(t, side)
        self._act(t)
        if side is not None:
            torch.cuda.current_stream(self.dev).wait_stream(side)

    def play_steps(self, check: bool = False) -> None:
        """One horizon.  The first observation is the last next-observation of the previous horizon.  Afterwards the student's Philox
        offset (shared with the reset draws) moves past the horizon.  check=True reads the getup error word (one host synchronisation)
        and raises if some fall env found no free fall state."""
        self.obses[:, 0].copy_(self.obs_carry)
        if self.physics is None and self.refresh is None:
            self._run(("horizon", self.teacher_side), self._whole)
        else:
            for t in range(self.T):
                self._run(("reset", t), self._reset, t)
                if self.refresh is not None:
                    self.refresh(t, self.reset_ws)
                self._run(("act", t, self.teacher_side), self._act_segment, t)
                if self.physics is not None:
                    self.physics(t)
                self._run(("post", t), self._env_step, t)
        self.vae.advance_rng(self.T)
        if check:
            self.comp.check_getup_error()

    def first_observation(self) -> None:
        """Observation of the initial state (Humanoid.reset -> _compute_observations at start-up): fills `obs_carry`."""
        self.comp.step(obs_buf=self.obs_carry, rew_buf=self.rewards[0], **self._step_kw())
        self.reset_buf.zero_()
        self.terminate_buf.zero_()

    def evaluate(self, dataset, physics=None, auto_pmcp: bool = False, auto_pmcp_soft: bool = False, **kw):
        """`IMAmpAgent.eval` (im_amp.py:136-242) of the student over every clip of `dataset` (a MotionDatasetB200) on this driver's
        simulator tensors: z = the posterior mean, the decoder's action, no teacher.  Then every env is reset into training through
        the getup reset (training probabilities; recovery episodes on the envs the pass's last step terminated) and the optional PMCP
        update (env_im_vae.yaml: auto_pmcp_soft): `evaluation.EvalStepsB200` (`kw`: its poll_every / use_graphs / strict_eval /
        eval_body_ids).  The pass is `self.eval_steps` while it runs: `physics(t)` applies its `pd_tar` and may read its task-side
        state (`progress_buf`, `motion_start_times`, ...)."""
        from .evaluation import EvalStepsB200
        self.eval_steps = EvalStepsB200(self, physics=physics, **kw)
        return self.eval_steps.run(dataset, auto_pmcp=auto_pmcp, auto_pmcp_soft=auto_pmcp_soft)

    # ------------------------------------------------------------------ update
    def _update_mb(self, i: int, minibatch: int, update_obs_rms: bool) -> None:
        r0, r1 = i * minibatch, (i + 1) * minibatch
        rows = self.n * self.T
        self.vae.optimize_kin(self.obses.view(rows, -1)[r0:r1], self.kin_gt.view(rows, -1)[r0:r1], self.kin_progress.view(rows)[r0:r1],
                              update_obs_rms=update_obs_rms)

    def train_epoch(self, epoch_num: int, mini_epochs: int = 6, minibatch: int = 16384, update_obs_rms: bool = True) -> torch.Tensor:
        """The only_kin_loss update of one epoch (`train_epoch` -> `_optimize_kin`, amp_agent.py:771-849): `mini_epochs` passes over the
        horizon's experience in contiguous minibatches of `minibatch` rows (whole envs: a multiple of the horizon), one
        `PulseVAE.optimize_kin` per minibatch and `anneal(epoch_num)` after each, as `AMPAgentB200Mixin._optimize_kin` does.  Each
        minibatch index is one CUDA graph; the KL coefficient is a launch argument, so the graphs are captured anew when annealing
        changes it (once per epoch past epoch 2500).  Returns the device stats tensor [mini_epochs, minibatches, 8] (fp64): each
        minibatch's `PulseVAE.stats`; `PulseVAE.losses(minibatch)` reads out the last one."""
        rows = self.n * self.T
        if minibatch <= 0 or minibatch % self.T or rows % minibatch:
            raise _lib.PulseError(f"minibatch {minibatch} must be a multiple of the horizon {self.T} dividing {rows} rows")
        num_mb = rows // minibatch
        if self.mb_stats is None or self.mb_stats.shape != (mini_epochs, num_mb, self.vae.stats.numel()):
            self.mb_stats = torch.zeros(mini_epochs, num_mb, self.vae.stats.numel(), dtype=torch.float64, device=self.dev)
        for k in range(mini_epochs):
            for i in range(num_mb):
                kld = self.vae.kld_coefficient
                if kld != self._kld:
                    self._graphs = {key: g for key, g in self._graphs.items() if key[0] != "update"}
                    self._kld = kld
                self._run(("update", i, minibatch, update_obs_rms), self._update_mb, i, minibatch, update_obs_rms)
                self.mb_stats[k, i].copy_(self.vae.stats)
                self.vae.anneal(epoch_num)
        return self.mb_stats
