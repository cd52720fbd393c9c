"""The task-independent part of the latent-space rollout drivers (`ZTaskStepsB200`, `TerrainStepsB200`): the experience buffers, the
action half of a step (the policy's heads beside the frozen prior, `pulse_latent_post`, the decoder), the next values, the launch
schedules, `play_steps`, `finish` and the PPO update (`AMPAgent.play_steps` + `train_epoch`, phc/learning/amp_agent.py:341-439,
:462-548; `HumanoidZ.step -> step_z`, humanoid_z.py:157-173)."""
import ctypes as C
from typing import Callable, Optional

import torch

from . import _lib
from .rollout import GraphRunner, finish_returns

# the AMP row entry point per body layout (AmpBuffersB200.layout)
_AMP_ROW = {"smpl": "pulse_amp_obs_row", "smplx": "pulse_smplx_amp_obs_row"}


class LatentStepsB200(GraphRunner):
    """One horizon of a latent-space task per `play_steps()`.  A subclass supplies the task's pieces of a step:
         `_reset(t)`           the reset of the done envs (Philox draws keyed (reset_seed, env, t + the policy's device offset)), which
                               leaves the reset's workspace {'env_list', 'count', ...} in `reset_ws`;
         `_reset_obs(t)`       the observation of the reset envs into obses[:, t], then the task's `_reset_task`;
         `_pre_physics(dec, t)` what the step does with the decoder output `dec` [n, A] before the physics (PD targets into pd_tar, ...);
         `_env_step(t)`        the rollout step kernel (progress += 1, reward, reset, next observation) into obses[:, t+1] / obs_carry,
                               rewards[t], dones[t], reset_buf, terminate_buf;
         `first_observation()` the observation of the initial state into obs_carry.
    For every step t, in the reference's order: `_reset(t)`, the `refresh(t, ws)` hook if set, `_reset_obs(t)`; `get_action_values`
    (the policy's `heads_into`, actor beside critic, and beside both the frozen prior MLP on obses[:, t, :S] with the clamped self
    observation columns of the decoder operand: neither depends on the action); `pulse_latent_post` (a_z = mu + exp(logstd) eps into
    actions[:, t], neglogp[:, t], the de-normalised value into values[t] and z = prior_mu + a_z into the decoder operand; the latent
    tasks' configs have clip_actions False and `project_to_norm(.., "none")` is the identity, so a_z is neither clamped nor projected);
    the decoder MLP on [clamp(norm(s), +-5) | z] (HumanoidZ.compute_z_actions); `_pre_physics`; the caller's `physics(t)` hook;
    `_env_step(t)`; next_values[t] = critic(obses[:, t+1]) (1 - terminate) on the critic's second operand slot.
    S and A are the VAE's self-observation width and dof count (358 and 69 for SMPL, 778 and 153 for SMPL-X), E its latent size.
    With `vae=None` the driver runs the non-latent task trained by PPO from scratch (learning=ppo): the policy acts in the A dofs
    (E = A), `get_action_values` is the heads and `pulse_policy_post` (actions, neglogp, de-normalised value), and `_pre_physics`
    takes the sampled actions themselves; there is no prior, `pulse_latent_post`, decoder or side P.
    `finish()` then computes GAE, normalised advantages and value-normalised returns from the task reward alone (task_reward_w 1,
    disc_reward_w 0) and `train_epoch()` runs the PPO update.

    The AMP part (opt-in: `amp`, an AmpBuffersB200, given exactly when the policy has a discriminator).  The driver then keeps the
    horizon's AMP rows `amp_obs[n, T, steps * width]` and the reset's back-filled history `amp_init[n, steps, width]` with its fresh
    flags; after the step kernel of every step, on main, `pulse_amp_obs_row` writes amp_obs[:, t] = [current row | the first steps - 1
    rows of amp_obs[:, t-1]] (of the back-filled rows for envs reset at step t: _init_amp_obs + _update_hist_amp_obs,
    humanoid_amp.py:519-563, :622-630).  `finish()` mixes task_reward_w * r + disc_reward_w * disc.rewards(amp_obs) (the discriminator
    forward pass is skipped at disc_reward_w 0); `train_epoch()` fetches amp_batch_size new demo rows, draws the demo and replay samples
    of the whole horizon (only the first amp_minibatch_size rows of each minibatch are gathered), passes amp = (amp_obs rows, replay
    rows, demo rows) at each minibatch's row offset to `train_minibatch` -- the discriminator's gradients share the actor / critic
    gradient-norm clip -- and stores the horizon's rows into the replay ring after the last mini-epoch; all of it graph-captured.
    Memory at 8192 envs, T = 32, 10 x 196 floats: amp_obs 2.06 GB, each 200 000-row ring 1.57 GB, each gathered sample 0.51 GB.  With
    the SMPL-X rows (10 x 465 floats): amp_obs n * 32 * 4650 * 4 B (0.91 GB at 1536 envs, 4.9 GB at 8192), the bf16 discriminator
    operand n * 32 * 4672 * 2 B (0.46 GB, 2.4 GB), each 200 000-row ring 3.72 GB.

    The experience buffers are env-major (`obses[n, T, W]`, `actions[n, T, E]`, `mus[n, T, E]`, `neglogp[n, T]`; `adv[n*T]`, `ret[n*T]`), so
    a minibatch is a contiguous row range; `values`, `next_values` [T, n, 1], `rewards`, `dones` [T, n] are time-major as GAE reads them.

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
       clear `terminate_buf`: the step kernel rewrites it for every env each step and nothing reads it in between.  The AMP row of step
       t runs on main after the step kernel(t): reset(t+1) rewrites the body state and the fresh flags it reads, and main's order keeps
       it before.
       With `physics` / `refresh` hooks the steps run as graph segments between the hook calls (reset | act | post), each with the same
       forks joined inside the segment.  `use_graphs=False` runs the same entry points on one stream in the order above.
       No ATen elementwise op, boolean-mask index or host synchronisation is inside the loop."""

    def _setup(self, task, reset, policy, vae, sim: dict, horizon: int, obs_width: int, pd_offset: Optional[torch.Tensor],
               pd_scale: Optional[torch.Tensor], pd_freeze: Optional[torch.Tensor], use_graphs: bool, gamma: float, tau: float,
               reset_seed: int, amp=None, task_reward_w: float = 1.0, disc_reward_w: float = 0.0) -> None:
        """The buffers and state every driver shares; the subclass calls it after its checks."""
        self.task, self.reset, self.policy, self.vae, self.sim, self.T = task, reset, policy, vae, sim, int(horizon)
        self.dev = policy.device
        self.lib = _lib.load()
        n = self.n
        # the policy acts in the latent (E) with a VAE, in the dof space (A) without one
        E, A = (vae.E, vae.A) if vae is not None else (policy.A, policy.A)
        T, W, dev = self.T, int(obs_width), self.dev
        self.dofs = A
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
        self.physics: Optional[Callable[[int], None]] = None           # physics(t): between the pre-physics work and the step kernel
        self.refresh: Optional[Callable[[int, dict], None]] = None     # refresh(t, ws): after the reset, before the reset envs' observation
        self.reset_ws = None
        self.z_actions = None          # the decoder's output of the last step, fp32 [n, A] (a reused workspace); None without a VAE
        self._streams = None
        self.amp, self.task_w, self.disc_w = amp, float(task_reward_w), float(disc_reward_w)
        if amp is None and (self.task_w != 1.0 or self.disc_w != 0.0):
            raise _lib.PulseError("task_reward_w / disc_reward_w mix in the discriminator reward: they need the AMP part (amp=AmpBuffersB200)")
        if amp is not None:
            if T < 2:
                raise _lib.PulseError("the AMP part needs a horizon of at least 2 steps (each AMP row shifts the previous step's row)")
            if policy.disc.size != amp.row_floats:
                raise _lib.PulseError(f"the discriminator reads {policy.disc.size} floats, the AMP rows have {amp.num_steps} x {amp.amp_width}")
            self.amp_obs = z(n, T, amp.row_floats)
            self.amp_init, self.amp_fresh = z(n, amp.num_steps, amp.amp_width), z(n, dtype=torch.int32)
            self.amp_x, self._amp_bufs = None, {}

    # ------------------------------------------------------------------ the task's pieces (subclass)
    def _reset(self, t: int) -> None:
        raise NotImplementedError

    def _reset_obs(self, t: int) -> None:
        raise NotImplementedError

    def _pre_physics(self, dec: torch.Tensor, t: int) -> None:
        raise NotImplementedError

    def _env_step(self, t: int) -> None:
        raise NotImplementedError

    def first_observation(self) -> None:
        raise NotImplementedError

    # ------------------------------------------------------------------ the shared pieces of one step
    def _launch(self, name: str, *args) -> None:
        with torch.cuda.device(self.dev):
            _lib.check(getattr(self.lib, name)(*args, _lib.current_stream(self.dev)), name)

    def _act(self, t: int, side_a=None, side_p=None) -> None:
        """get_action_values (amp_agent.py:359-378), HumanoidZ.compute_z_actions (humanoid_z.py:75-155) and the task's pre-physics work.
        Without a VAE (the dof-space baseline): the heads, `pulse_policy_post` (sample, neglogp, value) and the pre-physics work on the
        sampled actions, which are the dof actions (Humanoid.step -> pre_physics_step)."""
        pol, vae, n = self.policy, self.vae, self.n
        obs, mus = self.obses[:, t], self.mus[:, t]
        actions, neglogp, values = self.actions[:, t], self.neglogp[:, t], self.values[t]
        if vae is None:
            pol.act_into(obs, actions=actions, neglogp=neglogp, mus=mus, values=values, rng_step=t, side=side_a)
            self._pre_physics(actions, t)
            return
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

    def _amp_row(self, t: int) -> None:
        """The AMP row of step t (humanoid_amp.py:194-210, :622-667; amp_agent.py:385) into amp_obs[:, t], by the AMP part's body layout."""
        s, amp = self.sim, self.amp
        prev = self.amp_obs[:, t - 1] if t > 0 else self.amp_obs[:, self.T - 1]
        out = self.amp_obs[:, t]
        a = _lib.AmpRowArgs(body_state=s["body_state"].data_ptr(), body_env_stride=s["body_state"].stride(0), dof_pos=s["dof_pos"].data_ptr(),
                            dof_vel=s["dof_vel"].data_ptr(), dof_env_stride=s["dof_pos"].stride(0), dof_elem_stride=s["dof_pos"].stride(1),
                            prev=prev.data_ptr(), ld_prev=prev.stride(0), out=out.data_ptr(), ld_out=out.stride(0), num_steps=amp.num_steps,
                            fresh=self.amp_fresh.data_ptr(), fresh_rows=self.amp_init.data_ptr(), amp_width=amp.amp_width,
                            remove_base_rot=int(not amp.upright))
        self._launch(_AMP_ROW[amp.layout], C.byref(a), self.n)

    def _amp_start(self) -> None:
        """The AMP history of the initial state, for `first_observation`: the current AMP row in every history row of every env
        (_init_amp_obs_default, humanoid_amp.py:530-533), so that the first horizon's rows carry no zero history.  The reference builds
        the start-up history through its state init; with Random / Start it takes the history from the motion instead."""
        if self.amp is None:
            return
        W = self.amp.amp_width
        self._amp_row(self.T - 1)                                    # amp_obs[:, T-1, :W] = the current row (history from amp_obs[:, T-2])
        self.amp_init.copy_(self.amp_obs[:, self.T - 1, :W].unsqueeze(1).expand_as(self.amp_init))
        self.amp_obs[:, self.T - 1].copy_(self.amp_init.view(self.n, -1))
        self.amp_fresh.zero_()

    def _step(self, t: int) -> None:
        """The step kernel(t), then the AMP row of step t."""
        self._env_step(t)
        if self.amp is not None:
            self._amp_row(t)

    def _next_obs(self, t: int) -> torch.Tensor:
        return self.obses[:, t + 1] if t + 1 < self.T else self.obs_carry

    def _next_values(self, t: int, after_normalize=None) -> None:
        """`next_vals = _eval_critic(obs); next_vals *= 1 - terminated` (amp_agent.py:396-398), on the critic's second operand slot."""
        self.policy.critic_values_into(self._next_obs(t), self.next_values[t].view(-1), terminate=self.terminate_buf, slot=1,
                                       after_normalize=after_normalize)

    def _sides(self):
        """(A, P, B); no side P without a VAE (there is no prior to run)."""
        if self._streams is None:
            mk = lambda: torch.cuda.Stream(self.dev)
            self._streams = (mk(), mk() if self.vae is not None else None, mk())
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
            self._step(t)
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
            if self.amp is not None:
                self._amp_row(t)                                     # on main, beside B's next values, before reset(t+1)
        main.wait_stream(B)

    def _act_segment(self, t: int) -> None:
        self._reset_obs(t)
        self._act(t, *self._sides()[:2])

    def _post_segment(self, t: int) -> None:
        self._step(t)
        self._next_values(t)

    def play_steps(self) -> None:
        """One horizon.  The first observation is the last next-observation of the previous horizon.  Afterwards the policy's Philox
        offset (shared with the reset and task draws) moves past the horizon."""
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

    # ------------------------------------------------------------------ after the horizon
    def finish(self) -> None:
        """GAE + returns, advantage normalisation and value / return normalisation (`rollout.finish_returns`) of the mixed reward
        task_reward_w * r + disc_reward_w * disc_r (`_combine_rewards`, amp_agent.py:1011-1025); without the AMP part the task reward
        alone (task_reward_w 1, disc_reward_w 0)."""
        mb_rewards = self.rewards.unsqueeze(-1)
        if self.amp is not None:
            n, T = self.n, self.T
            if self.task_w != 1.0:
                mb_rewards = self.task_w * mb_rewards
            if self.disc_w != 0.0:                                   # disc_reward_w 0 adds 0 x a finite reward: the pass is skipped
                if self.amp_x is None:
                    from .nets import pad_k
                    self.amp_x = torch.zeros(n * T, pad_k(self.amp.row_floats), device=self.dev, dtype=torch.bfloat16)
                disc_r = self.policy.disc.rewards(self.amp_obs.view(n * T, -1), self.amp_x)      # env-major [n*T, 1]
                mb_rewards = mb_rewards + self.disc_w * disc_r.view(n, T).t().unsqueeze(-1)
        finish_returns(self.policy, self.dones, self.values, mb_rewards, self.next_values, self.adv, self.ret, self.gamma, self.tau)

    def _amp_batches(self, mb: int):
        """The gathered demo / replay samples of one epoch: [rows / mb * take, steps * width] each (a reused workspace)."""
        rows, amp = self.n * self.T, self.amp
        take = min(amp.minibatch_size, mb)
        if mb not in self._amp_bufs:
            z = lambda: torch.zeros(rows // mb * take, amp.row_floats, device=self.dev)
            self._amp_bufs[mb] = (z(), z())
        return take, self._amp_bufs[mb]

    def _amp_prelude(self, mb: int) -> None:
        """`_update_amp_demos`, then the demo sample and the replay sample (or the agent's rows) of train_epoch (amp_agent.py:476-484)."""
        amp, rows = self.amp, self.n * self.T
        _, (demo, replay) = self._amp_batches(mb)
        amp.update_demos()
        amp.sample(amp.demo, rows, mb, demo)
        amp.sample(amp.replay, rows, mb, replay, fallback=self.amp_obs.view(rows, -1))

    def _amp_store(self) -> None:
        self.amp.store_replay(self.amp_obs.view(self.n * self.T, -1))

    def _update_mb(self, i: int, mb: int) -> None:
        r0, r1 = i * mb, (i + 1) * mb
        rows = self.n * self.T
        amp = None
        if self.amp is not None:                             # amp_agent.py:621-628: the first amp_minibatch_size rows of each batch
            take, (demo, replay) = self._amp_batches(mb)
            amp = (self.amp_obs.view(rows, -1)[r0:r0 + take], replay[i * take:(i + 1) * take], demo[i * take:(i + 1) * take])
        self.policy.train_minibatch(self.obses.view(rows, -1)[r0:r1], self.actions.view(rows, -1)[r0:r1], self.neglogp.view(rows)[r0:r1],
                                    self.adv[r0:r1], self.ret[r0:r1], old_mu=self.mus.view(rows, -1)[r0:r1], amp=amp)

    def train_epoch(self, mini_epochs: int = 6, minibatch: int = 16384) -> torch.Tensor:
        """The PPO update of one epoch (`train_epoch` -> `calc_gradients`, amp_agent.py:462-548, :605-760; the discriminator term with
        the AMP part, see the class docstring): `mini_epochs` passes over the horizon's experience in contiguous minibatches of min(minibatch, n*T) rows, one
        `train_minibatch` each with old_mu = mus; every minibatch index is one CUDA graph.  Returns the policy's stats tensor,
        accumulated over the epoch (cleared at its start)."""
        rows = self.n * self.T
        mb = min(int(minibatch), rows)
        if mb <= 0 or rows % mb:
            raise _lib.PulseError(f"minibatch {minibatch} must divide the {rows} rows of a horizon")
        self.policy.reset_stats()
        if self.amp is not None:
            self._run(("amp_prelude", mb), self._amp_prelude, mb)
        for _ in range(mini_epochs):
            for i in range(rows // mb):
                self._run(("update", i, mb), self._update_mb, i, mb)
        if self.amp is not None:
            self._run(("amp_store",), self._amp_store)       # _store_replay_amp_obs after the update (amp_agent.py:539)
        return self.policy.stats
