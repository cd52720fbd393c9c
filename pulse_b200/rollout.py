"""Rollout post-processing on the device: GAE / returns / advantage normalisation.

Host-side mirror of `CommonAgent.discount_values` (phc/learning/common_agent.py:493-505),
`mb_returns = mb_advs + mb_values` (amp_agent.py:427) and `_calc_advs` (:589-599).
"""
import ctypes as C
import os

import torch

from . import _lib


def discount_values(mb_fdones: torch.Tensor, mb_values: torch.Tensor, mb_rewards: torch.Tensor, mb_next_values: torch.Tensor,
                    gamma: float = 0.99, tau: float = 0.95, normalize_advantage: bool = False):
    """Inputs time-major [T,N] / [T,N,1] as in the rl_games ExperienceBuffer.

    Returns (advantages, returns) ENV-MAJOR flat [N*T] -- the `swap_and_flatten01` layout the PPO
    dataset slices minibatches from.  With normalize_advantage=True the advantages are additionally
    normalised over the whole batch ((A-mean)/(std+1e-8), unbiased std) as `_calc_advs` does.
    """
    lib = _lib.load()
    T, N = mb_fdones.shape[0], mb_fdones.shape[1]
    dev = mb_rewards.device
    flat = lambda x: x.reshape(T, N).to(torch.float32).contiguous()
    r, v, nv, d = flat(mb_rewards), flat(mb_values), flat(mb_next_values), flat(mb_fdones)
    adv = torch.empty(N * T, device=dev, dtype=torch.float32)
    ret = torch.empty(N * T, device=dev, dtype=torch.float32)
    stats = torch.zeros(2, device=dev, dtype=torch.float64)
    a = _lib.GaeArgs(rewards=r.data_ptr(), values=v.data_ptr(), next_values=nv.data_ptr(), fdones=d.data_ptr(), gamma=gamma, tau=tau,
                     advantages=adv.data_ptr(), returns=ret.data_ptr(), adv_sum=stats.data_ptr())
    with torch.cuda.device(dev):
        st = _lib.current_stream(dev)
        _lib.check(lib.pulse_gae(C.byref(a), T, N, st), "pulse_gae")
        if normalize_advantage:
            _lib.check(lib.pulse_normalize_advantages(adv.data_ptr(), stats.data_ptr(), N * T, st), "pulse_normalize_advantages")
    return adv, ret


def finish_returns(pol, dones: torch.Tensor, values: torch.Tensor, mb_rewards: torch.Tensor, next_values: torch.Tensor, adv_out: torch.Tensor,
                   ret_out: torch.Tensor, gamma: float, tau: float) -> None:
    """The end of `play_steps` + `prepare_dataset` shared by the rollout drivers: GAE + returns (common_agent.py:493-505) and advantage
    normalisation (:589-599) into `adv_out`, value / return normalisation in training mode into `ret_out` (prepare_dataset :372-374: each
    tensor is normalised with the statistics BEFORE its own merge, running_mean_std.py:69-109).  Inputs time-major [T, n(, 1)], outputs
    env-major flat [n*T]."""
    adv, ret = discount_values(dones, values, mb_rewards, next_values, gamma=gamma, tau=tau, normalize_advantage=True)
    adv_out.copy_(adv)
    if pol.value_rms is not None:
        pol.value_rms.update(values.view(-1, 1))                                 # values: normalised copy unused (clip_value False), stats merged
        ret_out.copy_(pol.value_rms.normalize_values(ret.view(-1, 1)).view(-1))  # returns see the statistics that include the values batch ...
        pol.value_rms.update(ret.view(-1, 1))                                    # ... and are merged afterwards
    else:
        ret_out.copy_(ret)


class GraphRunner:
    """CUDA-graph runner of the rollout drivers: `_run(key, fn, *args)` executes `fn` eagerly on its first use, captures it on its second
    use and replays it from then on; every graph shares one memory pool.  The subclass sets `dev`, `use_graphs`, `_graphs = {}` and
    `_pool = None`."""

    def _run(self, key, fn, *args):
        if not self.use_graphs:
            return fn(*args)
        g = self._graphs.get(key)
        if g is None:
            # first use: plain eager execution (lazy workspaces, one-time attribute calls).  The segments are NOT idempotent (progress
            # counters advance, reset / fresh flags are consumed), so nothing may run twice: the capture happens on the second use,
            # where it only records, and the replay that follows is that use's single execution.
            self._graphs[key] = False
            return fn(*args)
        if g is False:
            torch.cuda.synchronize(self.dev)
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self._pool):
                fn(*args)
            self._graphs[key] = g
        g.replay()


class PlayStepsB200(GraphRunner):
    """`AMPAgent.play_steps` (phc/learning/amp_agent.py:341-439) on the device: for every step of the horizon
         env_reset(done envs) -> get_action_values -> env step (post-physics compute) -> AMP observation -> next values,
    then the discriminator rewards / reward mix / GAE / value normalisation of `play_steps` + `prepare_dataset`
    (amp_agent.py:418-437, common_agent.py:357-398).  Every kernel writes straight into the ENV-MAJOR experience buffers
    (`obses[n, T, 934]`, ...: a PPO minibatch is a contiguous row range, there is no swap_and_flatten01 copy); no ATen elementwise op,
    no host synchronisation and no boolean-mask indexing is left inside the loop.  Physics is the caller's: `physics(t)` is invoked
    between the action and the post-physics compute (bench.py passes nothing -- Isaac Gym is not installable, BASELINE.md 3.4).

    `sim`: the simulator's tensors, read / written IN PLACE through their strides (Isaac Gym views):
        body_state [N,B>=24,13], root_states [N,13] view, dof_pos / dof_vel [N,69] views, dof_force [N,69], progress_buf,
        motion_ids, motion_start_times, motion_start_offset, global_offset, cycle_counter (+ optional contact_forces, actor_ids).
    Launch structure: the work between two env steps (AMP row + next values of step t-1, resets + actions of step t) is one CUDA-graph
    segment; with `single_graph` the whole horizon including the fused step kernels is ONE graph and the step kernel is timed through
    graph-safe events (`_lib.GraphEvent`)."""

    def __init__(self, comp, policy, sim: dict, horizon: int = 32, task_reward_w: float = 0.5, disc_reward_w: float = 0.5,
                 pd_offset: torch.Tensor = None, pd_scale: torch.Tensor = None, use_graphs: bool = True, single_graph: bool = False,
                 gamma: float = 0.99, tau: float = 0.95, reset_seed: int = 0, time_steps: bool = True):
        self.comp, self.policy, self.sim, self.T = comp, policy, sim, int(horizon)
        self.dev = comp.device
        n = self.n = int(sim["progress_buf"].shape[0])
        T, dev = self.T, self.dev
        z = lambda *s, **k: torch.zeros(*s, device=dev, **k)
        self.obses, self.obs_carry = z(n, T, 934), z(n, 934)
        self.actions, self.mus, self.neglogp = z(n, T, policy.A), z(n, T, policy.A), z(n, T)
        self.amp_obs = z(n, T, 1960)
        self.values, self.next_values = z(T, n, 1), z(T, n, 1)
        self.rewards, self.dones = z(T, n), z(T, n)
        self.reward_raw = z(n, 5)
        self.reset_buf, self.terminate_buf = z(n, dtype=torch.long), z(n, dtype=torch.long)
        self.amp_init, self.amp_fresh = z(n, 10, 196), z(n, dtype=torch.int32)
        self.pd_tar = z(n, policy.A)
        self.pd = (pd_offset if pd_offset is not None else z(policy.A), pd_scale if pd_scale is not None else torch.ones(policy.A, device=dev))
        self.adv, self.ret = z(n * T), z(n * T)
        self.task_w, self.disc_w, self.gamma, self.tau = task_reward_w, disc_reward_w, gamma, tau
        self.reset_seed = (int(reset_seed) * 0x9E3779B97F4A7C15 + 0x13198A2E03707344) & (2 ** 64 - 1)
        self.use_graphs, self.single_graph, self.time_steps = use_graphs, single_graph, time_steps
        self._graphs, self._pool = {}, None
        self.step_events = [(_lib.GraphEvent(), _lib.GraphEvent()) for _ in range(T)] if time_steps else None
        self.amp_x = None
        self.host_io = None            # bench.py's end-to-end arm: (upload(t), download(t)) callables
        self.physics = None
        # Independent pieces of a step run on a second stream (fork / join inside the captured segment): the AMP row beside the
        # next-value critic, the critic beside the actor.  At 2048 envs per rank (8 GPUs) every kernel of the step is latency-bound
        # so the step time is the length of the dependency chain.
        self.fork = os.environ.get("PULSE_ROLLOUT_FORK", "1") != "0"
        self.overlap = os.environ.get("PULSE_ROLLOUT_OVERLAP", "1") != "0"   # next values of step t beside reset / actor of step t+1 (_whole_overlapped)
        self._side = None
        self._side_b = None
        self.amp_with_step = n <= 4096      # _whole_overlapped: AMP row concurrently with the fused step kernel only where both are latency-bound

    # ------------------------------------------------------------------ the pieces of one step
    def _step_kw(self):
        s = self.sim
        return dict(body_state=s["body_state"], dof_vel=s["dof_vel"], dof_force=s["dof_force"], progress_buf=s["progress_buf"],
                    motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                    global_offset=s["global_offset"], cycle_counter=s.get("cycle_counter"), reward_raw=self.reward_raw,
                    reset_buf=self.reset_buf, terminate_buf=self.terminate_buf)

    def _reset_and_act(self, t: int) -> None:
        """`self.obs = self.env_reset(done_indices)` (amp_agent.py:352) + `get_action_values` + experience updates (:355-378) + PD targets."""
        s, pol = self.sim, self.policy
        self.comp.reset_envs(motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                             global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
                             dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=self.reset_buf, terminate_buf=self.terminate_buf,
                             cycle_counter=s.get("cycle_counter"), contact_forces=s.get("contact_forces"), amp_obs_buf=self.amp_init,
                             actor_ids=s.get("actor_ids"), seed=self.reset_seed, offset=t, offset_dev=pol.rng_offset, obs_buf=self.obses[:, t],
                             amp_fresh=self.amp_fresh)
        pol.act_into(self.obses[:, t], actions=self.actions[:, t], neglogp=self.neglogp[:, t], mus=self.mus[:, t], values=self.values[t],
                     pd=(self.pd[0], self.pd[1], self.pd_tar), rng_step=t, side=self._side_stream())

    def _side_stream(self):
        if not self.fork:
            return None
        if self._side is None:
            self._side = torch.cuda.Stream(self.dev)
        return self._side

    def _next_obs(self, t: int) -> torch.Tensor:
        return self.obses[:, t + 1] if t + 1 < self.T else self.obs_carry

    def _env_step(self, t: int) -> None:
        """post_physics_step (humanoid.py:1315-1346): progress += 1, reward, reset, next observation -- one fused launch."""
        ev = self.step_events[t] if self.step_events is not None else None
        if ev is not None:
            ev[0].record(self.dev)
        self.comp.step(obs_buf=self._next_obs(t), rew_buf=self.rewards[t], fdones_out=self.dones[t], advance=True, **self._step_kw())
        if ev is not None:
            ev[1].record(self.dev)

    def _after_step(self, t: int) -> None:
        """AMP observation row of step t (humanoid_amp.py:194-210, amp_agent.py:385) and next_values (:396-398)."""
        s = self.sim
        prev = self.amp_obs[:, t - 1] if t > 0 else self.amp_obs[:, self.T - 1]
        side = self._side_stream()
        main = torch.cuda.current_stream(self.dev)
        if side is not None:
            side.wait_stream(main)
        with torch.cuda.stream(side if side is not None else main):
            self.comp.amp_obs_row(body_state=s["body_state"], dof_pos=s["dof_pos"], dof_vel=s["dof_vel"], prev=prev, out=self.amp_obs[:, t],
                                  fresh=self.amp_fresh, fresh_rows=self.amp_init)
        self.policy.critic_values_into(self._next_obs(t), self.next_values[t].view(-1), terminate=self.terminate_buf)
        if side is not None:
            main.wait_stream(side)     # the reset of the next segment rewrites the state / flags the AMP row reads

    def _segment(self, t: int) -> None:
        """Everything between env step t-1 and env step t."""
        if t > 0:
            self._after_step(t - 1)
            if self.host_io is not None:
                self.host_io[1](t - 1)
        if t < self.T:
            if self.host_io is not None:
                self.host_io[0](t)
            self._reset_and_act(t)

    # ------------------------------------------------------------------ graphs
    def _whole_overlapped(self) -> None:
        """The horizon with the independent pieces of consecutive steps overlapped on three streams (single-graph mode, no host I/O):
             main    reset(t) -> obs of the reset envs -> normalise -> actor -> policy_post -> fused step kernel(t)
             side A  critic(obs t) beside the actor;  AMP row(t) beside the step kernel
             side B  next values of step t (normalise -> critic -> value_post) beside reset(t+1) / actor(t+1)
           Hazards, all expressed as stream dependencies inside the captured graph: reset(t+1) rewrites the body state and the AMP
           `fresh` flags the AMP row(t) reads (main waits for A); the observation of the reset envs overwrites rows of obses[:, t+1]
           that B's normalise reads (main waits for the event B records after it); the step kernel(t+1) rewrites `terminate_buf` that
           B's value_post reads (main waits for B).  The reset does not clear `terminate_buf` here (the step kernel rewrites it for
           every env each step; nothing else reads it in between).  At 2048 envs per rank the step is a chain of latency-bound
           launches."""
        s, pol, T = self.sim, self.policy, self.T
        main = torch.cuda.current_stream(self.dev)
        A = self._side_stream()
        if self._side_b is None:
            self._side_b = torch.cuda.Stream(self.dev)
        B = self._side_b
        norm_done = None
        for t in range(T):
            if t > 0:
                main.wait_stream(A)                                  # AMP row(t-1) has read the pre-reset state
            ws = self.comp.reset_envs(motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                                      global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
                                      dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=self.reset_buf, terminate_buf=None,
                                      cycle_counter=s.get("cycle_counter"), contact_forces=s.get("contact_forces"), amp_obs_buf=self.amp_init,
                                      actor_ids=s.get("actor_ids"), seed=self.reset_seed, offset=t, offset_dev=pol.rng_offset, obs_buf=None,
                                      amp_fresh=self.amp_fresh)
            if norm_done is not None:
                main.wait_event(norm_done)                           # B has read obses[:, t]
            self.comp.step(body_state=s["body_state"], progress_buf=s["progress_buf"], motion_ids=s["motion_ids"],
                           motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"],
                           obs_buf=self.obses[:, t], env_ids=ws["env_list"][:self.n], env_count=ws["count"], flags=_lib.STEP_OBS)
            pol.act_into(self.obses[:, t], actions=self.actions[:, t], neglogp=self.neglogp[:, t], mus=self.mus[:, t], values=self.values[t],
                         pd=(self.pd[0], self.pd[1], self.pd_tar), rng_step=t, side=A)
            def amp_row():
                A.wait_stream(main)
                with torch.cuda.stream(A):
                    prev = self.amp_obs[:, t - 1] if t > 0 else self.amp_obs[:, T - 1]
                    self.comp.amp_obs_row(body_state=s["body_state"], dof_pos=s["dof_pos"], dof_vel=s["dof_vel"], prev=prev, out=self.amp_obs[:, t],
                                          fresh=self.amp_fresh, fresh_rows=self.amp_init)
            if self.amp_with_step:
                amp_row()                                            # beside the step kernel: both are latency-bound at small env counts
            if t > 0:
                main.wait_stream(B)                                  # value_post(t-1) has read terminate_buf
            self._env_step(t)
            if not self.amp_with_step:
                amp_row()                                            # large env counts: two HBM-bound kernels gain nothing from sharing the GPU
            B.wait_stream(main)
            with torch.cuda.stream(B):
                norm_done = torch.cuda.Event()
                self.policy.critic_values_into(self._next_obs(t), self.next_values[t].view(-1), terminate=self.terminate_buf, slot=1,
                                               after_normalize=lambda ev=norm_done: ev.record(B))
        main.wait_stream(A)
        main.wait_stream(B)

    def _whole(self) -> None:
        if self.fork and self.overlap and self.host_io is None and self.physics is None:
            return self._whole_overlapped()
        for t in range(self.T):
            self._segment(t)
            if self.physics is not None:
                self.physics(t)
            self._env_step(t)
        self._segment(self.T)

    def play_steps(self) -> None:
        """One horizon.  The first observation of the iteration is the last next-observation of the previous one."""
        self.obses[:, 0].copy_(self.obs_carry)
        io = self.host_io is not None
        if self.single_graph and self.physics is None:
            self._run(("rollout", io), self._whole)
        else:
            for t in range(self.T):
                self._run(("seg", t, io), self._segment, t)
                if self.physics is not None:
                    self.physics(t)
                self._env_step(t)
            self._run(("seg", self.T, io), self._segment, self.T)

    def first_observation(self) -> None:
        """Observation of the initial state (Humanoid.reset -> _compute_observations at start-up): fills `obs_carry`."""
        kw = self._step_kw()
        self.comp.step(obs_buf=self.obs_carry, rew_buf=self.rewards[0], **kw)
        self.reset_buf.zero_()
        self.terminate_buf.zero_()

    def step_kernel_ms(self):
        """Live durations of the fused step kernel launches of the LAST horizon (graph-safe events)."""
        return [a.elapsed_ms(b) for a, b in self.step_events] if self.step_events is not None else []

    def evaluate(self, dataset, physics=None, auto_pmcp: bool = False, auto_pmcp_soft: bool = False, **kw):
        """`IMAmpAgent.eval` (im_amp.py:136-242) of this policy over every clip of `dataset` (a MotionDatasetB200) on this driver's
        simulator tensors, then every env reset into training and the optional PMCP update: `evaluation.EvalStepsB200` (`kw`: its
        poll_every / use_graphs / strict_eval / eval_body_ids).  The pass is `self.eval_steps` while it runs: `physics(t)` applies
        its `pd_tar` and may read its task-side state (`progress_buf`, `motion_start_times`, ...)."""
        from .evaluation import EvalStepsB200
        self.eval_steps = EvalStepsB200(self, physics=physics, **kw)
        return self.eval_steps.run(dataset, auto_pmcp=auto_pmcp, auto_pmcp_soft=auto_pmcp_soft)

    # ------------------------------------------------------------------ after the horizon
    def finish(self) -> None:
        """Discriminator rewards over the whole horizon (amp_agent.py:422-424, :1027-1041), `_combine_rewards` (:1011-1025), GAE +
        returns (common_agent.py:493-505), advantage normalisation (:589-599), value / return normalisation in training mode
        (prepare_dataset :372-374: each tensor is normalised with the statistics BEFORE its own merge, running_mean_std.py:69-109)."""
        pol, n, T = self.policy, self.n, self.T
        if pol.disc is not None:
            if self.amp_x is None:
                from .nets import pad_k
                self.amp_x = torch.zeros(T * n, pad_k(1960), device=self.dev, dtype=torch.bfloat16)
            disc_r = pol.disc.rewards(self.amp_obs.view(n * T, 1960), self.amp_x)                    # env-major [n*T, 1]
            mb_rewards = self.task_w * self.rewards.unsqueeze(-1) + self.disc_w * disc_r.view(n, T).t().unsqueeze(-1)
        else:
            mb_rewards = self.rewards.unsqueeze(-1)
        finish_returns(pol, self.dones, self.values, mb_rewards, self.next_values, self.adv, self.ret, self.gamma, self.tau)
        pol.advance_rng(T)
