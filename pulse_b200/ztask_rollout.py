"""The latent-space tasks' training iteration on the device (BASELINE config C5): the rollout of HumanoidReachZ / HumanoidSpeedZ /
HumanoidStrikeZ with the frozen PULSE prior + decoder, device resets and the latent policy's PPO update (`AMPAgent.play_steps` +
`train_epoch`, phc/learning/amp_agent.py:341-439; `HumanoidAMPTask` resets, humanoid_amp_task.py:57-76; `HumanoidZ.step -> step_z`,
humanoid_z.py:157-173; pulse_z_task.yaml)."""
import ctypes as C
from typing import Callable, Optional

import torch

from . import _lib
from .rollout import GraphRunner, finish_returns

_KINDS = {_lib.ZTASK_REACH: "reach", _lib.ZTASK_SPEED: "speed", _lib.ZTASK_STRIKE: "strike"}
_WIDTHS = {"reach": 361, "speed": 361, "strike": 373}
SIM_KEYS = ("body_state", "root_states", "dof_pos", "dof_vel", "progress_buf", "sampled_motion_ids", "motion_start_times")
STRIKE_KEYS = ("target_states", "tar_contact_forces")


def check_pieces(task, reset, policy, vae) -> str:
    """The task kind ("reach" / "speed" / "strike") after checking that the step object, the reset, the latent policy and the frozen
    VAE belong together; raises PulseError otherwise."""
    kind = _KINDS.get(getattr(task, "kind", None))
    if kind is None:
        raise _lib.PulseError("ZTaskStepsB200: task must be a ReachTaskB200, SpeedTaskB200 or StrikeTaskB200")
    if getattr(reset, "kind", None) != kind:
        raise _lib.PulseError(f"ZTaskStepsB200: the reset serves {getattr(reset, 'kind', None)!r}, the task is {kind!r}")
    W = _WIDTHS[kind]
    if int(task.obs_size) != W or int(policy.obs_size) != W:
        raise _lib.PulseError(f"ZTaskStepsB200: the {kind} observation has {W} floats, the task writes {task.obs_size} and the policy reads {policy.obs_size}")
    if int(policy.A) != int(vae.E):
        raise _lib.PulseError(f"ZTaskStepsB200: the policy acts in {policy.A} dimensions, the VAE's latent has {vae.E}")
    if int(vae.S) != 358 or int(vae.A) != 69:
        raise _lib.PulseError(f"ZTaskStepsB200: the decoder must map the 358-float self observation to 69 dof targets, not {vae.S} -> {vae.A}")
    if getattr(policy, "disc", None) is not None:
        raise _lib.PulseError("ZTaskStepsB200: the discriminator is not part of this driver (task reward only); build the policy without it")
    return kind


class ZTaskStepsB200(GraphRunner):
    """One horizon of a latent-space task per `play_steps()`.  For every step t, in the reference's order:
         1. reset of the done envs (`ZTaskResetB200.reset_envs`, Philox draws keyed (reset_seed, env, t + the policy's device offset)),
            the `refresh(t, ws)` hook if set, the list observation of the reset envs into obses[:, t], then `reset_task` (reach, speed);
         2. `get_action_values`: the policy's normalise, actor beside critic; beside both, the frozen prior MLP on obses[:, t, :358] and
            the clamped self-observation columns of the decoder operand (neither depends on the action);
         3. `pulse_latent_post`: a_z = mu + exp(logstd) eps into actions[:, t], neglogp[:, t], the de-normalised value into values[t]
            and z = prior_mu + a_z into the decoder operand.  pulse_z_task.yaml has clip_actions False and `project_to_norm(.., "none")`
            is the identity, so a_z is neither clamped nor projected;
         4. the decoder MLP on [clamp(norm(s), +-5) | z]  (HumanoidZ.compute_z_actions, K20);
         5. `pulse_ztask_pre_physics`: PD targets into pd_tar, prev_root_pos (speed, strike), `_update_task` of the due envs (reach, speed);
         6. the caller's `physics(t)` hook;
         7. the rollout step kernel (progress += 1, reward, reset, next observation) into obses[:, t+1] / obs_carry, rewards[t], dones[t],
            reset_buf, terminate_buf;
         8. next_values[t] = critic(obses[:, t+1]) (1 - terminate).
    `finish()` then computes GAE, normalised advantages and value-normalised returns from the task reward alone (task_reward_w 1,
    disc_reward_w 0, pulse_z_task.yaml:90-91) and `train_epoch()` runs the PPO update.

    The experience buffers are env-major (`obses[n, T, W]`, `actions[n, T, E]`, `mus[n, T, E]`, `neglogp[n, T]`; `adv[n*T]`, `ret[n*T]`), so
    a minibatch is a contiguous row range; `values`, `next_values` [T, n, 1], `rewards`, `dones` [T, n] are time-major as GAE reads them.

    `task`: the ReachTaskB200 / SpeedTaskB200 / StrikeTaskB200 whose targets, change steps and termination settings the steps use.
    `reset`: the ZTaskResetB200 of the same kind.  `policy`: PPOPolicy(obs_size=task.obs_size, num_actions=vae.E, ...) without
    discriminator.  `vae`: PulseVAE(with_critic=False) holding the frozen prior, decoder and the checkpoint's obs_rms.  `sim`: the
    simulator's tensors, read and written in place through their strides: body_state, root_states, dof_pos, dof_vel, progress_buf,
    sampled_motion_ids, motion_start_times; optional contact_forces, actor_ids, dof_force (the speed task's power term); strike:
    target_states, tar_contact_forces and optional tar_actor_ids.

    Launch structure.  With no hooks the horizon is ONE CUDA graph over four streams:
         main    reset(t) -> obs of the reset envs -> reset_task -> normalise -> actor -> latent_post -> decoder -> pre_physics -> step kernel(t)
         side A  critic(obs t) beside the actor
         side P  prior operands + prior MLP(obs t) beside actor and critic
         side B  next values of step t (normalise -> critic -> value_post) beside reset(t+1) / actor(t+1)
       Hazards, all stream dependencies inside the captured graph: P starts after the observation of the reset envs (it reads obses[:, t]
       and rewrites the decoder operand's self columns, which decoder(t-1) on main has read by then); latent_post waits for A (value) and
       P (prior mean, decoder operand); the observation of the reset envs overwrites rows of obses[:, t+1] that B's normalise reads (main
       waits for the event B records after it); the step kernel(t+1) rewrites `terminate_buf` that B's value_post reads (main waits for B);
       B starts after the step kernel(t).  A and B use separate critic operands and workspaces (slot 0 / slot 1).  The reset does not
       clear `terminate_buf`: the step kernel rewrites it for every env each step and nothing reads it in between.
       With `physics` / `refresh` hooks the steps run as graph segments between the hook calls (reset | act | post), each with the same
       forks joined inside the segment.  `use_graphs=False` runs the same entry points on one stream in the order of the list above.
       No ATen elementwise op, boolean-mask index or host synchronisation is inside the loop.

    Out of scope: the discriminator (the reference still trains it here with disc_coef 5 although disc_reward_w is 0; leaving it out does
    not change the reward, but it removes the discriminator's gradients from the shared gradient-norm clip, so the reset is called
    without an AMP buffer); multi-GPU; the smplx humanoid; Default / Hybrid state init; the power_usage_reward terms the step kernels
    exclude."""

    def __init__(self, task, reset, policy, vae, sim: dict, horizon: int = 32, pd_offset: Optional[torch.Tensor] = None,
                 pd_scale: Optional[torch.Tensor] = None, pd_freeze: Optional[torch.Tensor] = None, use_graphs: bool = True,
                 gamma: float = 0.99, tau: float = 0.95, reset_seed: int = 0):
        self.kind = check_pieces(task, reset, policy, vae)
        missing = [k for k in SIM_KEYS + (STRIKE_KEYS if self.kind == "strike" else ()) if k not in sim]
        if missing:
            raise _lib.PulseError(f"ZTaskStepsB200: sim lacks {missing}")
        self.task, self.reset, self.policy, self.vae, self.sim, self.T = task, reset, policy, vae, sim, int(horizon)
        self.dev = policy.device
        self.lib = _lib.load()
        n = self.n = int(sim["progress_buf"].shape[0])
        if n != task.num_envs:
            raise _lib.PulseError(f"ZTaskStepsB200: sim has {n} envs, the task {task.num_envs}")
        T, W, E, A, dev = self.T, task.obs_size, vae.E, vae.A, self.dev
        z = lambda *s, **k: torch.zeros(*s, device=dev, **k)
        self.obses, self.obs_carry = z(n, T, W), z(n, W)
        self.actions, self.mus, self.neglogp = z(n, T, E), z(n, T, E), z(n, T)
        self.values, self.next_values = z(T, n, 1), z(T, n, 1)
        self.rewards, self.dones = z(T, n), z(T, n)
        self.reset_buf, self.terminate_buf = z(n, dtype=torch.long), z(n, dtype=torch.long)
        self.adv, self.ret = z(n * T), z(n * T)
        self.pd_tar = z(n, A)
        self.pd = (pd_offset if pd_offset is not None else z(A), pd_scale if pd_scale is not None else torch.ones(A, device=dev))
        if pd_freeze is not None and (pd_freeze.dtype != torch.uint8 or pd_freeze.numel() != A):
            raise _lib.PulseError(f"pd_freeze must be uint8 [{A}]")
        self.pd_freeze = pd_freeze
        self.gamma, self.tau = gamma, tau
        self.reset_seed = (int(reset_seed) * 0x9E3779B97F4A7C15 + 0x13198A2E03707344) & (2 ** 64 - 1)
        self.use_graphs = use_graphs
        self._graphs, self._pool = {}, None
        self.physics: Optional[Callable[[int], None]] = None           # physics(t): between the pre-physics kernel and the step kernel
        self.refresh: Optional[Callable[[int, dict], None]] = None     # refresh(t, ws): after the reset, before the reset envs' observation
        self.reset_ws = None
        self.z_actions = None          # the decoder's output of the last step, fp32 [n, 69] (a reused workspace)
        self._streams = None

    # ------------------------------------------------------------------ the pieces of one step
    def _step_args(self, obs: torch.Tensor, rew: torch.Tensor):
        """The task's step arguments with the outputs pointed at experience slices and the driver's reset / terminate words."""
        s, task = self.sim, self.task
        if self.kind == "reach":
            a = task._step_args(s["body_state"], s["progress_buf"], s.get("contact_forces"))
        else:
            a = task._args(s["body_state"], s["progress_buf"], s.get("contact_forces"))
            if self.kind == "speed":
                a.tar_speed = task._tar_speed.data_ptr()
                if task.power_reward:
                    if s.get("dof_force") is None:
                        raise _lib.PulseError("the speed task's power_reward needs sim['dof_force']")
                    a.dof_force, a.dof_force_stride, a.power_coefficient = s["dof_force"].data_ptr(), s["dof_force"].stride(0), task.power_coefficient
                    a.dof_vel, a.dof_env_stride, a.dof_elem_stride = s["dof_vel"].data_ptr(), s["dof_vel"].stride(0), s["dof_vel"].stride(1)
            else:
                a.target_states, a.target_env_stride = s["target_states"].data_ptr(), s["target_states"].stride(0)
                a.tar_contact_forces, a.tar_contact_env_stride = s["tar_contact_forces"].data_ptr(), s["tar_contact_forces"].stride(0)
        a.obs_buf, a.obs_stride, a.rew_buf = obs.data_ptr(), obs.stride(0), rew.data_ptr()
        a.reset_buf, a.terminate_buf = self.reset_buf.data_ptr(), self.terminate_buf.data_ptr()
        return a

    def _launch(self, name: str, *args) -> None:
        with torch.cuda.device(self.dev):
            _lib.check(getattr(self.lib, name)(*args, _lib.current_stream(self.dev)), name)

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
            reset_buf=self.reset_buf, contact_forces=s.get("contact_forces"), amp_obs_buf=None, actor_ids=s.get("actor_ids"),
            target_states=s["target_states"] if strike else None, tar_actor_ids=s.get("tar_actor_ids") if strike else None,
            seed=self.reset_seed, offset=t, offset_dev=self.policy.rng_offset)

    def _reset_obs(self, t: int) -> None:
        """`_compute_observations(env_ids)` of the reset envs into obses[:, t], then `_reset_task` (humanoid_amp_task.py:66-76)."""
        ws = self.reset_ws
        a = self._step_args(self.obses[:, t], self.rewards[t])
        self._launch("pulse_reach_obs_list" if self.kind == "reach" else "pulse_ztask_obs_list", C.byref(a), ws["env_list"].data_ptr(),
                     ws["count"].data_ptr(), self.n)
        if self.kind != "strike":
            self.reset.reset_task(progress_buf=self.sim["progress_buf"], seed=self.reset_seed, offset=t, offset_dev=self.policy.rng_offset,
                                  **self._task_kw())

    def _act(self, t: int, side_a=None, side_p=None) -> None:
        """get_action_values (amp_agent.py:359-378), HumanoidZ.compute_z_actions (humanoid_z.py:75-155) and pre_physics_step."""
        pol, vae, n = self.policy, self.vae, self.n
        obs, mus = self.obses[:, t], self.mus[:, t]
        main = torch.cuda.current_stream(self.dev)
        if side_p is not None:
            side_p.wait_stream(main)
            with torch.cuda.stream(side_p):
                prior_head, dec_in = vae.z_prior(obs)
        else:
            prior_head, dec_in = vae.z_prior(obs)
        value = pol.heads_into(obs, mus=mus, side=side_a)
        if side_p is not None:
            main.wait_stream(side_p)
        actions, neglogp, values = self.actions[:, t], self.neglogp[:, t], self.values[t]
        rms = pol.value_rms
        a = _lib.LatentPostArgs(mu=mus.data_ptr(), ld_mu=mus.stride(0), logstd=pol.logstd.data_ptr(), seed=pol.rng_seed,
                                rng_offset=pol.rng_offset.data_ptr(), rng_step=t, latent=vae.E, actions=actions.data_ptr(),
                                ld_actions=actions.stride(0), neglogp=neglogp.data_ptr(), ld_neglogp=neglogp.stride(0),
                                value=value.data_ptr(), ld_value=value.stride(0), values_out=values.data_ptr(), ld_values=values.stride(0),
                                prior_mu=prior_head.data_ptr(), ld_prior=prior_head.stride(0), z_bf16=dec_in.data_ptr(), ld_z=dec_in.stride(0))
        if rms is not None:
            a.value_mean, a.value_var, a.value_eps = rms.running_mean.data_ptr(), rms.running_var.data_ptr(), rms.eps
        self._launch("pulse_latent_post", C.byref(a), n)
        self.z_actions = dec = vae.dec.forward(dec_in)
        self._pre_physics(dec, t)

    def _pre_physics(self, dec: torch.Tensor, t: int, rand: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None) -> None:
        """`pulse_ztask_pre_physics` on the decoder output `dec` [n, 69]; `rand` / `steps` inject the `_update_task` draws per env."""
        s, task, kind = self.sim, self.task, self.kind
        p = _lib.ZTaskPrePhysicsArgs(kind=task.kind, dofs=self.vae.A, action=dec.data_ptr(), ld_action=dec.stride(0), pd_offset=self.pd[0].data_ptr(),
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

    def _next_obs(self, t: int) -> torch.Tensor:
        return self.obses[:, t + 1] if t + 1 < self.T else self.obs_carry

    def _env_step(self, t: int) -> None:
        """post_physics_step (humanoid.py:1315-1346): one fused launch."""
        a = self._step_args(self._next_obs(t), self.rewards[t])
        self._launch("pulse_reach_rollout_step" if self.kind == "reach" else "pulse_ztask_rollout_step", C.byref(a), self.dones[t].data_ptr(), self.n)

    def _next_values(self, t: int, after_normalize=None) -> None:
        """`next_vals = _eval_critic(obs); next_vals *= 1 - terminated` (amp_agent.py:396-398), on the critic's second operand slot."""
        self.policy.critic_values_into(self._next_obs(t), self.next_values[t].view(-1), terminate=self.terminate_buf, slot=1,
                                       after_normalize=after_normalize)

    def _sides(self):
        if self._streams is None:
            self._streams = tuple(torch.cuda.Stream(self.dev) for _ in range(3))
        return self._streams

    # ------------------------------------------------------------------ schedules
    def _sequential(self) -> None:
        """The horizon on one stream, hooks included, in the order of the class docstring."""
        for t in range(self.T):
            self._reset(t)
            if self.refresh is not None:
                self.refresh(t, self.reset_ws)
            self._reset_obs(t)
            self._act(t)
            if self.physics is not None:
                self.physics(t)
            self._env_step(t)
            self._next_values(t)

    def _whole_overlapped(self) -> None:
        """The horizon without hooks over main + sides A, P, B (hazards: class docstring)."""
        main = torch.cuda.current_stream(self.dev)
        A, P, B = self._sides()
        norm_done = None
        for t in range(self.T):
            self._reset(t)
            if norm_done is not None:
                main.wait_event(norm_done)                           # B has read obses[:, t]
            self._reset_obs(t)
            self._act(t, A, P)
            if t > 0:
                main.wait_stream(B)                                  # value_post(t-1) has read terminate_buf
            self._env_step(t)
            B.wait_stream(main)
            with torch.cuda.stream(B):
                norm_done = torch.cuda.Event()
                self._next_values(t, after_normalize=lambda ev=norm_done: ev.record(B))
        main.wait_stream(B)

    def _act_segment(self, t: int) -> None:
        self._reset_obs(t)
        self._act(t, *self._sides()[:2])

    def _post_segment(self, t: int) -> None:
        self._env_step(t)
        self._next_values(t)

    def play_steps(self) -> None:
        """One horizon.  The first observation is the last next-observation of the previous horizon.  Afterwards the policy's Philox
        offset (shared with the reset and `_update_task` draws) moves past the horizon."""
        self.obses[:, 0].copy_(self.obs_carry)
        if not self.use_graphs:
            self._sequential()
        elif self.physics is None and self.refresh is None:
            self._run(("horizon",), self._whole_overlapped)
        else:
            for t in range(self.T):
                self._run(("reset", t), self._reset, t)
                if self.refresh is not None:
                    self.refresh(t, self.reset_ws)
                self._run(("act", t), self._act_segment, t)
                if self.physics is not None:
                    self.physics(t)
                self._run(("post", t), self._post_segment, t)
        self.policy.advance_rng(self.T)

    def first_observation(self) -> None:
        """Observation of the initial state (Humanoid.reset -> _compute_observations at start-up): fills `obs_carry`."""
        a = self._step_args(self.obs_carry, self.rewards[0])
        self._launch("pulse_reach_step" if self.kind == "reach" else "pulse_ztask_step", C.byref(a), self.n)
        self.reset_buf.zero_()
        self.terminate_buf.zero_()

    # ------------------------------------------------------------------ after the horizon
    def finish(self) -> None:
        """GAE + returns, advantage normalisation and value / return normalisation (`rollout.finish_returns`) from the task reward alone:
        task_reward_w 1, disc_reward_w 0 (pulse_z_task.yaml:90-91; `_combine_rewards`, amp_agent.py:1011-1025)."""
        finish_returns(self.policy, self.dones, self.values, self.rewards.unsqueeze(-1), self.next_values, self.adv, self.ret, self.gamma, self.tau)

    def _update_mb(self, i: int, mb: int) -> None:
        r0, r1 = i * mb, (i + 1) * mb
        rows = self.n * self.T
        self.policy.train_minibatch(self.obses.view(rows, -1)[r0:r1], self.actions.view(rows, -1)[r0:r1], self.neglogp.view(rows)[r0:r1],
                                    self.adv[r0:r1], self.ret[r0:r1], old_mu=self.mus.view(rows, -1)[r0:r1])

    def train_epoch(self, mini_epochs: int = 6, minibatch: int = 16384) -> torch.Tensor:
        """The PPO update of one epoch (`train_epoch` -> `calc_gradients`, amp_agent.py:462-548, :605-760, without the discriminator
        term): `mini_epochs` passes over the horizon's experience in contiguous minibatches of min(minibatch, n*T) rows, one
        `PPOPolicy.train_minibatch` each with old_mu = mus; every minibatch index is one CUDA graph.  Returns the policy's stats
        tensor, accumulated over the epoch (cleared at its start)."""
        rows = self.n * self.T
        mb = min(int(minibatch), rows)
        if mb <= 0 or rows % mb:
            raise _lib.PulseError(f"minibatch {minibatch} must divide the {rows} rows of a horizon")
        self.policy.reset_stats()
        for _ in range(mini_epochs):
            for i in range(rows // mb):
                self._run(("update", i, mb), self._update_mb, i, mb)
        return self.policy.stats
