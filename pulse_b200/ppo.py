"""PPO actor / critic on the GPU: host-side mirror of the agent-side arithmetic of
`phc.learning.common_agent.CommonAgent` / `amp_agent.AMPAgent` for the continuous-action 'amp' network
(separate actor and critic MLPs, fixed log-std; im.yaml:13-42):

  get_action_values   common_agent.py:262-288  -> PPOPolicy.act
  _eval_critic        common_agent.py:552-562  -> PPOPolicy.critic_values
  calc_gradients      amp_agent.py:605-760 (actor / critic / bound losses, grad-norm clip, Adam) -> PPOPolicy.train_minibatch
  _preproc_obs        amp_agent.py:586-603 + RunningMeanStd (running_mean_std.py:69-109)          -> RunningMeanStdB200

The discriminator branch of calc_gradients (AMP style loss with gradient penalty, amp_agent.py:895-952) lives in
`pulse_b200/amp.py` and shares this class's flat parameter / gradient buffers (one optimizer, one norm clip).  Multi-GPU: gradients are all-reduced (average) over torch.distributed's NCCL
communicator once per minibatch on the flat gradient buffer, replacing Horovod's DistributedOptimizer
(amp_agent.py:735-742).
"""
import ctypes as C
import math
import os
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .nets import MLP, FlatParams, normalize_to_bf16, pad8, pad_k


class RunningMeanStdB200:
    """phc/utils/running_mean_std.py:9-109 with fp64 statistics kept on the device."""

    def __init__(self, size: int, device, epsilon: float = 1e-5):
        self.size, self.device, self.eps = size, device, epsilon
        self.running_mean = torch.zeros(size, dtype=torch.float64, device=device)
        self.running_var = torch.ones(size, dtype=torch.float64, device=device)
        self.count = torch.ones((), dtype=torch.float64, device=device)
        self._sums = torch.zeros(2 * size, dtype=torch.float64, device=device)
        self.frozen = False
        self.pad_one = 0.0     # 1.0: the first pad column of the normalised bf16 operand is the "ones" column of a bias-augmented first layer
        self.mean_f32 = torch.zeros(size, dtype=torch.float32, device=device)
        self.rstd_f32 = torch.ones(size, dtype=torch.float32, device=device)
        self._refresh()

    def _refresh(self):
        # in place: the buffers' addresses stay fixed, so normalise / update sequences can be captured in CUDA graphs
        self.mean_f32.copy_(self.running_mean)
        self.rstd_f32.copy_(1.0 / torch.sqrt(self.running_var.float() + self.eps))

    def _merge(self, lib, n: int) -> None:
        _lib.check(lib.pulse_rms_merge(self._sums.data_ptr(), n, self.size, self.running_mean.data_ptr(), self.running_var.data_ptr(),
                                       self.count.data_ptr(), self.eps, self.mean_f32.data_ptr(), self.rstd_f32.data_ptr(),
                                       _lib.current_stream(self.device)), "pulse_rms_merge")     # leaves _sums zeroed

    def update(self, x: torch.Tensor) -> None:
        """Training-mode statistics update (:96-107): Welford merge with the batch mean / unbiased variance."""
        if self.frozen:
            return
        lib = _lib.load()
        with torch.cuda.device(self.device):
            _lib.check(lib.pulse_column_moments(x.data_ptr(), x.stride(0), x.shape[0], self.size, self._sums.data_ptr(),
                                                _lib.current_stream(self.device)), "pulse_column_moments")
            self._merge(lib, x.shape[0])

    def normalize_update(self, x: torch.Tensor, out: torch.Tensor) -> None:
        """forward() in training mode (:91-107): normalise with the CURRENT statistics, then merge this batch -- one
        pass over x (pulse_normalize_moments) + the merge launch."""
        if self.frozen:
            return self.normalize_into(x, out)
        lib = _lib.load()
        with torch.cuda.device(self.device):
            _lib.check(lib.pulse_normalize_moments(x.data_ptr(), x.stride(0), x.shape[0], self.size, self.mean_f32.data_ptr(),
                                                   self.rstd_f32.data_ptr(), out.data_ptr(), out.stride(0), self._sums.data_ptr(), self.pad_one,
                                                   _lib.current_stream(self.device)), "pulse_normalize_moments")
            self._merge(lib, x.shape[0])

    def normalize_into(self, x: torch.Tensor, out: torch.Tensor, out_t: Optional[torch.Tensor] = None) -> None:
        normalize_to_bf16(x, self.mean_f32, self.rstd_f32, out, out_t, pad_one=self.pad_one)

    def normalize_split(self, x: torch.Tensor, self_cols: int, p: torch.Tensor, p_off: int, t: torch.Tensor, update: bool) -> None:
        """forward() of an observation [self | task] into two bias-augmented operands in one pass (pulse_normalize_split):
        p[:, p_off:] = [self | 1 | 0...], t = [task | 1 | 0...].  update=True (training mode, unless frozen) merges the batch afterwards."""
        if x.dtype != torch.float32 or x.stride(1) != 1 or x.shape[1] != self.size:
            raise _lib.PulseError("normalize_split: x must be fp32 [rows, size] with contiguous rows")
        lib = _lib.load()
        upd = update and not self.frozen
        with torch.cuda.device(self.device):
            _lib.check(lib.pulse_normalize_split(x.data_ptr(), x.stride(0), x.shape[0], self.size, self_cols, self.mean_f32.data_ptr(),
                                                 self.rstd_f32.data_ptr(), p.data_ptr(), p.stride(0), p_off, t.data_ptr(), t.stride(0),
                                                 self._sums.data_ptr() if upd else None, _lib.current_stream(self.device)),
                       "pulse_normalize_split")
            if upd:
                self._merge(lib, x.shape[0])

    def unnormalize(self, y: torch.Tensor) -> torch.Tensor:
        """forward(unnorm=True) (:84-87): clamp to +-5 then scale back (value de-normalisation)."""
        return torch.clamp(y, -5.0, 5.0) * torch.sqrt(self.running_var.float() + self.eps) + self.running_mean.float()

    def normalize_values(self, x: torch.Tensor) -> torch.Tensor:
        return torch.clamp((x - self.running_mean.float()) / torch.sqrt(self.running_var.float() + self.eps), -5.0, 5.0)


class PPOPolicy:
    def __init__(self, obs_size: int = 934, num_actions: int = 69, units: Sequence[int] = (1024, 512), act: str = "relu",
                 logstd: float = -2.9, device="cuda:0", seed: int = 0, lr: float = 2e-5, e_clip: float = 0.2, critic_coef: float = 5.0,
                 bounds_coef: float = 10.0, grad_norm: float = 50.0, normalize_value: bool = True, with_disc: bool = False,
                 amp_obs_size: int = 1960, disc_units: Sequence[int] = (1024, 512)):
        self.device = torch.device(device)
        self.obs_size, self.A = obs_size, num_actions
        self.lr, self.e_clip, self.critic_coef, self.bounds_coef, self.grad_norm = lr, e_clip, critic_coef, bounds_coef, grad_norm
        self.flat = FlatParams(self.device)
        self._build_nets(obs_size, units, act)
        self.disc = None
        if with_disc:  # one optimizer / one grad-norm clip over actor + critic + discriminator, as in the reference
            from .amp import AmpDiscriminator
            self.disc = AmpDiscriminator(self.flat, amp_obs_size, disc_units)
        self.flat.finalize()
        gen = torch.Generator(device=self.device).manual_seed(seed)
        for net in self._policy_nets():
            net.init_default(gen)
        if self.disc is not None:
            self.disc.mlp.init_default(gen)
        self.logstd = torch.full((num_actions,), logstd, device=self.device)  # fixed_sigma, const_initializer (im.yaml:21-25)
        self.obs_rms = RunningMeanStdB200(obs_size, self.device)
        self.obs_rms.pad_one = 1.0             # the normalised observation operand carries the first layers' ones column
        self.value_rms = RunningMeanStdB200(1, self.device) if normalize_value else None
        self.Kp = self.actor.Kp0
        self._bufs: Dict[tuple, dict] = {}
        self.stats = torch.zeros(6, dtype=torch.float64, device=self.device)
        self.lib = _lib.load()
        self._side = None
        self.rng_seed = (int(seed) * 0x9E3779B97F4A7C15 + 0x243F6A8885A308D3) & (2 ** 64 - 1)
        self.rng_offset = torch.zeros(1, dtype=torch.int64, device=self.device)    # uint64 counter read by the sampling kernel

    def _build_nets(self, obs_size: int, units: Sequence[int], act: str) -> None:
        # bias-augmented layers (nets.Dense): bias add and bias gradients are done by the tensor cores, the epilogues carry neither
        self.actor = MLP(self.flat, obs_size, units, self.A, act, aug=True)
        self.critic = MLP(self.flat, obs_size, units, 1, act, aug=True)

    def _policy_nets(self):
        """The nets besides the discriminator, in initialisation order."""
        return (self.actor, self.critic)

    # ------------------------------------------------------------------ buffers
    def _buf(self, M: int, train: bool):
        key = (M, train)
        if key not in self._bufs:
            dev = self.device
            b = {}
            if train:
                b["x2"] = torch.zeros(2, M, self.Kp, device=dev, dtype=torch.bfloat16)     # two operand slots (prepare_inputs)
                Ap = pad8(self.A)
                b.update(dmu=torch.zeros(M, Ap, device=dev, dtype=torch.bfloat16), dv=torch.zeros(M, 8, device=dev, dtype=torch.bfloat16))
            else:
                b.update(x=torch.zeros(M, self.Kp, device=dev, dtype=torch.bfloat16), actions=torch.zeros(M, self.A, device=dev),
                         neglogp=torch.zeros(M, device=dev))
            self._bufs[key] = b
        return self._bufs[key]

    def _normalize_eval(self, obs: torch.Tensor, b: dict) -> None:
        """Evaluation-mode input of the actor / critic: b['x'] <- normalised obs."""
        self.obs_rms.normalize_into(obs, b["x"])

    # ------------------------------------------------------------------ rollout side
    def act(self, obs: torch.Tensor, eps: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """get_action_values (common_agent.py:262-288): normalise obs, actor + critic forward, sample, neglogp.
        `eps` lets a test inject the standard-normal draw."""
        M = obs.shape[0]
        b = self._buf(M, False)
        self._normalize_eval(obs, b)
        mu = self.actor.forward(b["x"])
        value = self.critic.forward(b["x"])
        if eps is None:
            eps = torch.randn(M, self.A, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_gaussian_sample(mu.data_ptr(), mu.stride(0), eps.data_ptr(), self.logstd.data_ptr(), M, self.A,
                                                      b["actions"].data_ptr(), b["neglogp"].data_ptr(), _lib.current_stream(self.device)),
                       "pulse_gaussian_sample")
        values = self.value_rms.unnormalize(value) if self.value_rms is not None else value
        return {"actions": b["actions"], "neglogpacs": b["neglogp"], "values": values, "mus": mu,
                "sigmas": torch.exp(self.logstd).expand(M, self.A)}

    def act_into(self, obs: torch.Tensor, *, actions: torch.Tensor, neglogp: torch.Tensor, mus: torch.Tensor, values: Optional[torch.Tensor] = None,
                 pd: Optional[tuple] = None, eps: Optional[torch.Tensor] = None, rng_step: int = 0, side=None) -> None:
        """get_action_values (common_agent.py:262-288) + the experience-buffer updates of play_steps (amp_agent.py:361-378) + the PD
        targets of pre_physics_step (humanoid.py:1222-1257) with NO intermediate copies: the actor head GEMM writes `mus` (a
        [M, A] slice of the experience buffer, any row stride), `pulse_policy_post` draws the noise in-kernel (Philox; `eps`
        injects it for tests) and writes actions / neglogp / de-normalised values / PD targets through (pointer, stride).
        pd = (offset [A], scale [A], out [M, A]).  `side`: a second CUDA stream -- the critic's forward pass then runs beside the
        actor's (at the per-rank env counts of a multi-GPU run neither fills the GPU)."""
        M = obs.shape[0]
        value = self.heads_into(obs, mus=mus, with_value=values is not None, side=side)
        a = _lib.PolicyPostArgs(mu=mus.data_ptr(), ld_mu=mus.stride(0), logstd=self.logstd.data_ptr(), seed=self.rng_seed,
                                rng_offset=self.rng_offset.data_ptr(), rng_step=int(rng_step), num_actions=self.A,
                                actions=actions.data_ptr(), ld_actions=actions.stride(0), neglogp=neglogp.data_ptr(), ld_neglogp=neglogp.stride(0))
        if eps is not None:
            a.eps, a.ld_eps = eps.data_ptr(), eps.stride(0)
        if values is not None:
            a.value, a.ld_value, a.values_out, a.ld_values = value.data_ptr(), value.stride(0), values.data_ptr(), values.stride(0)
            if self.value_rms is not None:
                a.value_mean, a.value_var, a.value_eps = self.value_rms.running_mean.data_ptr(), self.value_rms.running_var.data_ptr(), self.value_rms.eps
        if pd is not None:
            a.pd_offset, a.pd_scale, a.pd_targets, a.ld_pd = pd[0].data_ptr(), pd[1].data_ptr(), pd[2].data_ptr(), pd[2].stride(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_policy_post(C.byref(a), M, _lib.current_stream(self.device)), "pulse_policy_post")

    def heads_into(self, obs: torch.Tensor, *, mus: torch.Tensor, with_value: bool = True, side=None) -> Optional[torch.Tensor]:
        """The network half of get_action_values: normalise `obs`, the actor head into `mus` ([M, A] slice, any row stride) and, with
        `with_value`, the critic; returns its NORMALISED value [M, 1] (a reused workspace) or None.  `side`: the critic runs on that
        stream beside the actor and is joined before returning."""
        b = self._buf(obs.shape[0], False)
        self._normalize_eval(obs, b)
        if side is not None and with_value:              # actor | critic on two streams (fork / join: still one CUDA-graph segment)
            main = torch.cuda.current_stream(self.device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                value = self.critic.forward(b["x"])
            self.actor.forward(b["x"], out=mus)
            main.wait_stream(side)
            return value
        self.actor.forward(b["x"], out=mus)
        return self.critic.forward(b["x"]) if with_value else None

    def critic_values_into(self, obs: torch.Tensor, out: torch.Tensor, terminate: Optional[torch.Tensor] = None, slot: int = 0,
                           after_normalize=None) -> None:
        """`next_vals = self._eval_critic(self.obs); next_vals *= (1.0 - terminated)` (amp_agent.py:396-398) into `out` ([M] / [M,1] view).
        `slot` 1: a second operand buffer / critic workspace, so that this evaluation may run on another stream beside `act_into`;
        `after_normalize()` is called once `obs` has been read (the caller records an event there: `obs` may be overwritten after it)."""
        M = obs.shape[0]
        b = self._buf(M, False)
        x = b["x"]
        if slot:
            if "x_next" not in b:
                b["x_next"] = torch.zeros_like(b["x"])
            x = b["x_next"]
        self.obs_rms.normalize_into(obs, x)
        if after_normalize is not None:
            after_normalize()
        self._value_post(self.critic.forward(x, slot=slot), terminate, out)

    def _value_post(self, value: torch.Tensor, terminate: Optional[torch.Tensor], out: torch.Tensor) -> None:
        """`pulse_value_post`: out = de-normalised `value` (* (1 - terminate) when given)."""
        rms = self.value_rms
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_value_post(value.data_ptr(), value.stride(0), rms.running_mean.data_ptr() if rms is not None else None,
                                                 rms.running_var.data_ptr() if rms is not None else None, rms.eps if rms is not None else 0.0,
                                                 _lib.ptr(terminate), out.data_ptr(), out.stride(0), value.shape[0], _lib.current_stream(self.device)),
                       "pulse_value_post")

    def advance_rng(self, steps: int) -> None:
        """Moves the device-side Philox offset past the `steps` draws of a rollout (keeps CUDA-graph replays statistically fresh)."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_bump_counter(self.rng_offset.data_ptr(), int(steps), _lib.current_stream(self.device)), "pulse_bump_counter")

    def _reducer(self, world_size: int):
        if world_size <= 1:
            return None
        if getattr(self, "_chain_reducer", None) is None:
            from .dist_utils import ChainReducer
            self._chain_reducer = ChainReducer(world_size, 3)
        return self._chain_reducer

    def reset_stats(self) -> None:
        """The loss statistics ACCUMULATE over train_minibatch calls (sum over rows; one mini-epoch's mean KL = stats[3] / rows seen):
        clear them where the reference starts a new list (amp_agent.py:496-505)."""
        self.stats.zero_()

    def sync_stats(self, world_size: int) -> None:
        """`hvd.sync_stats` once per epoch (common_agent.py:126-127) [3P-memory: HorovodWrapper averages every running-statistics
        tensor]: observation, value and AMP-input normalisers."""
        if world_size <= 1:
            return
        from .dist_utils import sync_running_stats
        for rms in (self.obs_rms, self.value_rms, self.disc.rms if self.disc is not None else None):
            if rms is not None:
                sync_running_stats(rms.running_mean, rms.running_var, rms.count, world_size)
                rms._refresh()

    def critic_values(self, obs: torch.Tensor) -> torch.Tensor:
        """_eval_critic (common_agent.py:552-562)."""
        M = obs.shape[0]
        b = self._buf(M, False)
        self._normalize_eval(obs, b)
        value = self.critic.forward(b["x"])
        return self.value_rms.unnormalize(value) if self.value_rms is not None else value

    # ------------------------------------------------------------------ update side
    def prepare_inputs(self, obs, amp=None, update_obs_rms: bool = True, slot: int = 0) -> None:
        """The weight-independent head of calc_gradients for one minibatch: observation normalisation in train mode (statistics
        BEFORE this batch, then merge it: running_mean_std.py:91-107) and `_preproc_amp_obs` of the three AMP batches, into
        operand slot `slot`.  train_minibatch(prefetch=...) runs it for the NEXT minibatch on a side stream, off the critical
        path (under the backward GEMMs, or under the gradient all-reduce on several GPUs)."""
        b = self._buf(obs.shape[0], True)
        if update_obs_rms:
            self.obs_rms.normalize_update(obs, b["x2"][slot])
        else:
            self.obs_rms.normalize_into(obs, b["x2"][slot])
        if amp is not None:
            self.disc.prepare_inputs(*amp, slot=slot)

    def train_minibatch(self, obs, actions, old_neglogp, advantages, returns, old_mu=None, update_obs_rms: bool = True,
                        world_size: int = 1, amp=None, keep_grads: bool = False, slot: int = 0, prepared: bool = False,
                        prefetch=None) -> torch.Tensor:
        """One calc_gradients step (amp_agent.py:605-760, PPO branch without the discriminator term).
        `returns` are already value-normalised (prepare_dataset, common_agent.py:372-374).  Returns the fp64
        stats tensor [sum a_loss, sum c_loss, sum b_loss, sum kl, clipped, sum neglogp], ACCUMULATED since reset_stats() (divide by the
        rows seen).
        `slot` / `prepared`: the normalised operands of this minibatch live in slot `slot`; `prepared=True` says prepare_inputs()
        already filled it.  `prefetch=(obs_next, amp_next)`: prepare_inputs() of the NEXT minibatch into slot `1 - slot` on a side
        stream (same order of running-statistics updates as the reference: batch i+1 after batch i)."""
        M = obs.shape[0]
        b = self._buf(M, True)
        # Three independent chains -- actor, critic, discriminator -- run on three streams (fork/join with events, so
        # the whole minibatch still captures into ONE CUDA graph): the persistent GEMMs of one chain fill the partial
        # last wave of another, and the HBM-bound normalise / moments / loss kernels overlap with tensor-core work.
        main = torch.cuda.current_stream(self.device)
        if self._side is None:
            self._side = (torch.cuda.Stream(self.device), torch.cuda.Stream(self.device), torch.cuda.Stream(self.device))
        _, s_disc, s_pref = self._side
        # where the next minibatch's input preparation is forked: under the NCCL all-reduce when there is one (it leaves most SMs idle);
        # at the start, under the GEMMs, on one GPU and with the peer-memory optimizer kernel (which occupies every SM while it runs)
        peer_step = self.flat.peer is not None and world_size > 1 and not keep_grads
        pref_at = os.environ.get("PULSE_PREFETCH_AT", "reduce" if (world_size > 1 and not peer_step) else "start") if prefetch is not None else None

        def fork_prefetch():
            s_pref.wait_stream(main)
            with torch.cuda.stream(s_pref):
                self.prepare_inputs(prefetch[0], prefetch[1], update_obs_rms, 1 - slot)

        self.flat.begin_backward()                                # weight / bias gradients are accumulated by bulk reductions / atomics
        reducer = self._reducer(world_size)                  # multi-GPU: every chain averages ITS gradient slice on its own stream
        # Reducing every chain's slice on its own stream ("chain") does not hide the collective: the persistent GEMMs own every SM and
        # walk a static tile schedule, so NCCL's CTAs either wait for a GEMM to drain or delay the CTAs of the next one -- the collective
        # is interleaved, not overlapped.  Default: one all-reduce; PULSE_GRAD_REDUCE=chain keeps the per-chain variant for experiments.
        single = reducer is not None and os.environ.get("PULSE_GRAD_REDUCE", "single") != "chain"
        if single:
            reducer = None
        # with a prefetch, this minibatch's AMP batches are normalised here, before the fork: the next minibatch's, on the prefetch stream,
        # merge into the same discriminator input statistics and must come after them
        amp_here = not prepared and prefetch is not None
        if not prepared:
            self.prepare_inputs(obs, amp if amp_here else None, update_obs_rms, slot)
        if pref_at == "start":
            fork_prefetch()
        if amp is not None:                                  # (agent, replay, demo) AMP observation batches: disc_coef * disc_loss
            s_disc.wait_stream(main)
            with torch.cuda.stream(s_disc):
                self.disc.loss_backward(*amp, slot=slot, prepared=prepared or amp_here)
                if reducer is not None:
                    d0, d1 = self.disc.mlp.param_span()
                    reducer.reduce(self.flat.grads[d0:d1], 2)
        mu, value = self._forward_train(b, slot)
        a = _lib.PpoLossArgs(
            mu=mu.data_ptr(), ld_mu=mu.stride(0), value=value.data_ptr(), ld_value=value.stride(0), actions=actions.data_ptr(),
            old_neglogp=old_neglogp.data_ptr(), advantages=advantages.data_ptr(), returns=returns.data_ptr(),
            old_mu=old_mu.data_ptr() if old_mu is not None else None, logstd=self.logstd.data_ptr(), num_actions=self.A,
            e_clip=self.e_clip, critic_coef=self.critic_coef, bounds_coef=self.bounds_coef,
            dmu=b["dmu"].data_ptr(), ld_dmu=b["dmu"].stride(0), dvalue=b["dv"].data_ptr(), ld_dv=b["dv"].stride(0),
            stats=self.stats.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_ppo_loss(C.byref(a), M, _lib.current_stream(self.device)), "pulse_ppo_loss")
        if pref_at == "loss":
            fork_prefetch()
        self._backward_train(b, M, reducer)
        if amp is not None:
            main.wait_stream(s_disc)
        if pref_at == "reduce":
            fork_prefetch()
        if peer_step:
            # one kernel per rank over NVLink peer memory: reduce-scatter of the gradients, norm clip, Adam on the rank's slice, push of
            # the new masters / bf16 operands to every rank (csrc/peer_adam.cu) -- no NCCL call on the data path
            self.flat.peer_adam_step(self.lr, max_norm=self.grad_norm)
        else:
            if single:
                from .dist_utils import average_gradients
                average_gradients(self.flat.grads, world_size)
            self.flat.adam_step(self.lr, max_norm=self.grad_norm, zero_grads=not keep_grads)  # also writes the bf16 operand mirror, clears the gradients
        if pref_at is not None:
            main.wait_stream(s_pref)
        return self.stats

    def _forward_train(self, b: dict, slot: int):
        """Training forward pass of the policy nets on operand slot `slot` of the minibatch buffers: (mu, value), fp32."""
        x = b["x2"][slot]
        main, s_critic = torch.cuda.current_stream(self.device), self._side[0]
        s_critic.wait_stream(main)
        with torch.cuda.stream(s_critic):
            value = self.critic.forward(x, train=True)
        mu = self.actor.forward(x, train=True)
        main.wait_stream(s_critic)
        return mu, value

    def _backward_train(self, b: dict, M: int, reducer) -> None:
        """Backward pass of the policy nets from the loss kernel's output gradients b['dmu'] / b['dv']; `reducer` (multi-GPU, per-chain
        gradient exchange) averages each net's gradient slice once it is complete."""
        main, s_critic = torch.cuda.current_stream(self.device), self._side[0]
        s_critic.wait_stream(main)
        with torch.cuda.stream(s_critic):
            self.critic.backward(b["dv"], M)
            if reducer is not None:
                c0, c1 = self.critic.param_span()
                reducer.reduce(self.flat.grads[c0:c1], 1)
        self.actor.backward(b["dmu"], M)
        if reducer is not None:
            a0, a1 = self.actor.param_span()
            reducer.reduce(self.flat.grads[a0:a1], 0)
        main.wait_stream(s_critic)

    # ------------------------------------------------------------------ checkpoint keys (rl_games layout)
    def _rms_pairs(self):
        """(checkpoint section, normaliser): A2CBase.get_stats_weights [rl_games] + AMPAgent.get_stats_weights (amp_agent.py:181-189)."""
        out = [("running_mean_std", self.obs_rms)]
        if self.value_rms is not None:
            out.append(("reward_mean_std", self.value_rms))
        if self.disc is not None:
            out.append(("amp_input_mean_std", self.disc.rms))
        return out

    def _named_layers(self):
        """(reference parameter prefix, Dense) in the order `ModelAMPContinuous.named_parameters()` yields them is NOT needed: every
        consumer goes by name."""
        out = []
        nets = [(self.actor, "actor_mlp", "mu"), (self.critic, "critic_mlp", "value")]
        if self.disc is not None:
            nets.append((self.disc.mlp, "_disc_mlp", "_disc_logits"))
        for mlp, prefix, head in nets:
            for i, l in enumerate(mlp.layers[:-1]):
                out.append((f"a2c_network.{prefix}.{2 * i}", l))
            out.append((f"a2c_network.{head}", mlp.layers[-1]))
        return out

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Model parameters under the reference's checkpoint keys (network_loader.py:81-99 reads them) + the three normalisers under
        `<section>.running_mean|running_var|count`."""
        sd = {}
        for name, l in self._named_layers():
            sd[name + ".weight"] = l.ref_weight()
            sd[name + ".bias"] = l.bias.clone()
        sd["a2c_network.sigma"] = self.logstd.clone()
        for sec, rms in self._rms_pairs():
            sd[f"{sec}.running_mean"], sd[f"{sec}.running_var"], sd[f"{sec}.count"] = rms.running_mean.clone(), rms.running_var.clone(), rms.count.clone()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        for name, l in self._named_layers():
            if name + ".weight" in sd:
                l.set_weights(sd[name + ".weight"].to(self.device), sd[name + ".bias"].to(self.device))
        if "a2c_network.sigma" in sd:
            self.logstd.copy_(sd["a2c_network.sigma"].to(self.device))
        for sec, rms in self._rms_pairs():
            if f"{sec}.running_mean" in sd:
                rms.running_mean.copy_(sd[f"{sec}.running_mean"].to(self.device).double().reshape(-1))
                rms.running_var.copy_(sd[f"{sec}.running_var"].to(self.device).double().reshape(-1))
                if f"{sec}.count" in sd:
                    rms.count.copy_(torch.as_tensor(sd[f"{sec}.count"]).to(self.device).double().reshape(()))
                rms._refresh()

    def optimizer_state(self, gather: bool = True) -> Dict[str, Dict[str, torch.Tensor]]:
        """torch.optim.Adam state per reference parameter name: {'exp_avg', 'exp_avg_sq'} in the parameter's shape, plus 'step'."""
        out = {}
        if gather:
            self.flat.gather_moments()  # peer mode keeps the moments sharded over the ranks (COLLECTIVE; no-op otherwise).  A caller that runs on
                                        # one rank only (rank-0 checkpointing) gathers at a point every rank reaches and passes gather=False
        step = self.flat.step.clone().float().reshape(())
        for name, l in self._named_layers():
            m, v = self.flat.view(l.w_idx, "exp_avg"), self.flat.view(l.w_idx, "exp_avg_sq")
            out[name + ".weight"] = {"exp_avg": l.ref_weight("exp_avg"), "exp_avg_sq": l.ref_weight("exp_avg_sq"), "step": step.clone()}
            if l.aug:
                out[name + ".bias"] = {"exp_avg": m[:, l.K].clone(), "exp_avg_sq": v[:, l.K].clone(), "step": step.clone()}
            else:
                out[name + ".bias"] = {"exp_avg": self.flat.view(l.b_idx, "exp_avg").clone(), "exp_avg_sq": self.flat.view(l.b_idx, "exp_avg_sq").clone(),
                                       "step": step.clone()}
        return out

    def load_optimizer_state(self, state: Dict[str, Dict[str, torch.Tensor]]) -> None:
        step = None
        for name, l in self._named_layers():
            for kind in ("weight", "bias"):
                st = state.get(f"{name}.{kind}")
                if st is None or "exp_avg" not in st:
                    continue
                m, v = self.flat.view(l.w_idx, "exp_avg"), self.flat.view(l.w_idx, "exp_avg_sq")
                if kind == "weight":
                    l.set_ref_weight("exp_avg", st["exp_avg"].to(self.device))
                    l.set_ref_weight("exp_avg_sq", st["exp_avg_sq"].to(self.device))
                elif l.aug:
                    m[:, l.K].copy_(st["exp_avg"].to(self.device))
                    v[:, l.K].copy_(st["exp_avg_sq"].to(self.device))
                else:
                    self.flat.view(l.b_idx, "exp_avg").copy_(st["exp_avg"].to(self.device))
                    self.flat.view(l.b_idx, "exp_avg_sq").copy_(st["exp_avg_sq"].to(self.device))
                step = st.get("step", step)
        if step is not None:
            self.flat.step.fill_(int(float(step)))
