"""PPO policy for the `amp_sept` network of the pedestrian terrain task (pulse_z_terrain.yaml): a task encoder shared by the actor and
the critic (`AMPSeptBuilder.Network`, phc/learning/amp_network_sept_builder.py).

Reference network.  obs = [self (S) | traj + heightmap (T)], normalised as a whole by the observation RunningMeanStd;
`eval_actor` / `eval_critic` each compute `task_out = _task_mlp(obs[:, S:])` (Linear+act after EVERY layer, _build_mlp) and feed
`cat([self_obs, task_out])` into their own MLP.  There is ONE `_task_mlp` (`separate: True` builds it twice; the second build replaces the
first), so its gradient is the sum of what the actor loss and the critic loss send back through it.

Device layout (operand columns, bf16):
    P [M, pad_k(E + S + 1)] = [task_out (E) | self (S) | 1 | 0...]    input of actor_mlp.0 and critic_mlp.0
    T [M, pad_k(T + 1)]     = [traj + heightmap (T) | 1 | 0...]       input of _task_mlp.0
One pass over the fp32 observations writes both (pulse_normalize_split).  The task net's top layer writes SiLU(.) straight into P[:, :E]
(the embedding goes first: column 0 is 16-byte aligned for the GEMM epilogue, column S is not).  The first layers of the actor and the
critic keep their weight columns in P's order; checkpoints and Adam moments are exchanged in the reference's [self | task_out] order
(Dense.ref_cols).

Backward.  The first layers of the actor and the critic are reserved back to back in the flat buffers, and their output gradients
(gated by SiLU') are the two column halves of ONE [M, 2 N0] buffer, so the embedding gradient of BOTH consumers is one dgrad GEMM over
the concatenated K:
    dEmb = SiLU'(pre_top) * ([dPre0_actor | dPre0_critic] . [W_a0[:, :E] ; W_c0[:, :E]])
the actor + critic sum happening in the GEMM's fp32 accumulator.  The task net's backward then runs from dEmb.
"""
import os
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .dense import gemm
from .nets import MLP, Dense, pad8
from .ppo import PPOPolicy


class SeptPolicy(PPOPolicy):
    def __init__(self, self_obs_size: int = 358, task_obs_size_detail: Optional[Dict[str, int]] = None, task_units: Sequence[int] = (512, 256),
                 units: Sequence[int] = (2048, 1024, 512), act: str = "silu", num_actions: int = 32, with_disc: bool = True,
                 task_act: Optional[str] = None, logstd: float = -1.0, **kw):
        detail = dict(task_obs_size_detail) if task_obs_size_detail is not None else {"traj": 20, "heightmap": 1024}
        if set(detail) != {"traj", "heightmap"}:
            raise _lib.PulseError(f"SeptPolicy covers task_obs_size_detail {{traj, heightmap}} only, got {sorted(detail)} "
                                  "(the 'people' PointNet branch and the velocity map are not built)")
        self.S = int(self_obs_size)
        self.task_in = int(detail["traj"]) + int(detail["heightmap"])
        self.task_units = tuple(int(u) for u in task_units)
        self.task_act = task_act or act
        self.E = self.task_units[-1]
        if self.task_act != "silu":
            raise _lib.PulseError(f"SeptPolicy: the task encoder's activation must be silu, got {self.task_act}")
        if self.S % 2 or self.task_in % 2 or self.E % 8:
            raise _lib.PulseError("SeptPolicy: the self and task observation sizes must be even and the task embedding a multiple of 8")
        super().__init__(obs_size=self.S + self.task_in, num_actions=num_actions, units=units, act=act, with_disc=with_disc, logstd=logstd, **kw)
        a0 = self.actor.layers[0]
        off = self.flat.offset(a0.w_idx)
        self._w0_cat = self.flat.params_bf16[off:off + 2 * a0.N * a0.Kp].view(2 * a0.N, a0.Kp)   # [W_a0 ; W_c0], bf16 operand mirror

    def _build_nets(self, obs_size: int, units: Sequence[int], act: str) -> None:
        flat, n_in = self.flat, self.E + self.S
        self.task = MLP(flat, self.task_in, self.task_units, None, self.task_act, aug=True)
        a0, c0 = Dense(flat, n_in, units[0], act, aug=True), Dense(flat, n_in, units[0], act, aug=True)
        if flat.offset(c0.w_idx) != flat.offset(a0.w_idx) + a0.N * a0.Kp:
            raise _lib.PulseError("SeptPolicy: the actor's and the critic's first layers must be adjacent in the flat buffers")
        a0.ref_cols = c0.ref_cols = torch.cat([torch.arange(self.E, n_in), torch.arange(0, self.E)])   # reference [self | emb] -> internal
        self.actor = MLP(flat, n_in, units, self.A, act, aug=True, first=a0)
        self.critic = MLP(flat, n_in, units, 1, act, aug=True, first=c0)

    def _policy_nets(self):
        return (self.task, self.actor, self.critic)

    # ------------------------------------------------------------------ buffers
    def _buf(self, M: int, train: bool):
        new = (M, train) not in self._bufs
        b = super()._buf(M, train)                # x / x2: the policy operand P (width = the actor's Kp0)
        if new:
            dev, bf = self.device, torch.bfloat16
            tw = self.task.Kp0
            if train:
                n0 = self.actor.layers[0].N
                b["t2"] = torch.zeros(2, M, tw, device=dev, dtype=bf)
                b["dpre0"] = torch.zeros(M, 2 * n0, device=dev, dtype=bf)      # [actor | critic] gradients w.r.t. the first layers' pre-activations
                b["demb"] = torch.zeros(M, pad8(self.E), device=dev, dtype=bf)
                self.actor.provide_dact0(M, b["dpre0"][:, :n0])
                self.critic.provide_dact0(M, b["dpre0"][:, n0:])
            else:
                b["t"] = torch.zeros(M, tw, device=dev, dtype=bf)
        return b

    # ------------------------------------------------------------------ rollout side
    def _normalize_eval(self, obs: torch.Tensor, b: dict) -> None:
        """b['x'] <- [embedding | normalised self | 1 | 0...]: normalise_split, then the task encoder into its first E columns.  Run
        once before the actor | critic fork of `heads_into`; both heads read the same operand."""
        self.obs_rms.normalize_split(obs, self.S, b["x"], self.E, b["t"], update=False)
        self.task.forward(b["t"], out=b["x"][:, :self.E])

    def critic_values_into(self, obs: torch.Tensor, out: torch.Tensor, terminate: Optional[torch.Tensor] = None, slot: int = 0,
                           after_normalize=None) -> None:
        """PPOPolicy.critic_values_into through the shared task encoder.  `slot` 1 uses operands of its own (x_next, t_next) and the
        slot-1 workspaces of the encoder and the critic, none of which `heads_into` touches on slot 0, so that it may run on another
        stream beside it; `after_normalize()` is called once `obs` has been read."""
        M = obs.shape[0]
        b = self._buf(M, False)
        x, t = b["x"], b["t"]
        if slot:
            if "x_next" not in b:
                b["x_next"], b["t_next"] = torch.zeros_like(b["x"]), torch.zeros_like(b["t"])
            x, t = b["x_next"], b["t_next"]
        self.obs_rms.normalize_split(obs, self.S, x, self.E, t, update=False)
        if after_normalize is not None:
            after_normalize()
        self.task.forward(t, out=x[:, :self.E], slot=slot)
        self._value_post(self.critic.forward(x, slot=slot), terminate, out)

    # ------------------------------------------------------------------ update side
    def _reducer(self, world_size: int):
        if world_size > 1 and os.environ.get("PULSE_GRAD_REDUCE", "single") == "chain":
            raise _lib.PulseError("SeptPolicy: PULSE_GRAD_REDUCE=chain is not supported (the shared task encoder's gradient is complete only "
                                  "after both the actor and the critic); use the default single exchange")
        return super()._reducer(world_size)

    def prepare_inputs(self, obs, amp=None, update_obs_rms: bool = True, slot: int = 0) -> None:
        b = self._buf(obs.shape[0], True)
        self.obs_rms.normalize_split(obs, self.S, b["x2"][slot], self.E, b["t2"][slot], update_obs_rms)
        if amp is not None:
            self.disc.prepare_inputs(*amp, slot=slot)

    def _forward_train(self, b: dict, slot: int):
        self.task.forward(b["t2"][slot], train=True, out=b["x2"][slot][:, :self.E])
        return super()._forward_train(b, slot)

    def _backward_train(self, b: dict, M: int, reducer) -> None:
        super()._backward_train(b, M, None)                 # reducer is None: chain exchange refused in _reducer
        gemm(b["dpre0"], self._w0_cat[:, :self.E], b_mn=True, gate=self.task.top_preact(M), gate_mode="silu", out=b["demb"])
        self.task.backward(b["demb"], M)

    # ------------------------------------------------------------------ checkpoint keys
    def _named_layers(self):
        return [(f"a2c_network._task_mlp.{2 * i}", l) for i, l in enumerate(self.task.layers)] + super()._named_layers()
