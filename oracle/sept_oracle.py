"""torch fp32 restatement of the `amp_sept` policy network and of its PPO + AMP loss (the pedestrian terrain task's agent).

  AMPSeptBuilder.Network.eval_actor / eval_critic / eval_task   phc/learning/amp_network_sept_builder.py:46-109
  calc_gradients total loss                                     phc/learning/amp_agent.py:691-711
      actor + critic_coef * critic + bounds_coef * bound + disc_coef * disc   (entropy_coef 0, clip_value False)

Parameters are a state dict under the reference's names without the `a2c_network.` prefix.  Runs on any device; the tests use it on
the CPU against tests/golden/sept.npz and on the GPU at production widths.
"""
from typing import Dict, List, Tuple

import torch

from . import pulse_oracle as po


def _stack(sd: Dict[str, torch.Tensor], prefix: str) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    ws, bs, i = [], [], 0
    while f"{prefix}.{i}.weight" in sd:
        ws.append(sd[f"{prefix}.{i}.weight"])
        bs.append(sd[f"{prefix}.{i}.bias"])
        i += 2
    return ws, bs


def eval_task(sd, obs: torch.Tensor, self_obs_size: int, act: str = "silu") -> torch.Tensor:
    """_task_mlp(obs[:, S:]): _build_mlp puts the activation after every layer, the last one included."""
    ws, bs = _stack(sd, "_task_mlp")
    return po.mlp_forward(obs[:, self_obs_size:], ws, bs, act)


def _trunk(sd, prefix: str, head: str, obs, self_obs_size: int, act: str) -> torch.Tensor:
    x = torch.cat([obs[:, :self_obs_size], eval_task(sd, obs, self_obs_size, act)], dim=-1)
    ws, bs = _stack(sd, prefix)
    return torch.nn.functional.linear(po.mlp_forward(x, ws, bs, act), sd[f"{head}.weight"], sd[f"{head}.bias"])


def eval_actor(sd, obs: torch.Tensor, self_obs_size: int, act: str = "silu") -> torch.Tensor:
    """mu of eval_actor (mu_activation None); sigma is the fixed `sigma` parameter."""
    return _trunk(sd, "actor_mlp", "mu", obs, self_obs_size, act)


def eval_critic(sd, obs: torch.Tensor, self_obs_size: int, act: str = "silu") -> torch.Tensor:
    return _trunk(sd, "critic_mlp", "value", obs, self_obs_size, act)


def eval_disc(sd, amp_obs: torch.Tensor) -> torch.Tensor:
    """AMPBuilder.Network.eval_disc: ReLU `_disc_mlp` + linear `_disc_logits`."""
    ws, bs = _stack(sd, "_disc_mlp")
    return torch.nn.functional.linear(po.mlp_forward(amp_obs, ws, bs, "relu"), sd["_disc_logits.weight"], sd["_disc_logits.bias"])


def total_loss(sd, obs, actions, old_neglogp, advantages, returns, amp=None, self_obs_size: int = 358, act: str = "silu",
               critic_coef: float = 5.0, bounds_coef: float = 10.0, disc_coef: float = 5.0) -> Dict[str, torch.Tensor]:
    """The calc_gradients loss on normalised observations `obs` and (if given) normalised AMP batches amp = (agent, replay, demo)."""
    mu = eval_actor(sd, obs, self_obs_size, act)
    value = eval_critic(sd, obs, self_obs_size, act)
    out = po.ppo_total_loss(mu, value[:, 0], old_neglogp, advantages, returns, actions, sd["sigma"], critic_coef=critic_coef, bounds_coef=bounds_coef)
    out.update(mu=mu, value=value)
    if amp is not None:
        w = [sd[f"_disc_mlp.{i}.weight"] for i in range(0, 2 * len(_stack(sd, "_disc_mlp")[0]), 2)] + [sd["_disc_logits.weight"]]
        d = po.disc_loss(lambda x: eval_disc(sd, x), amp[0], amp[1], amp[2], sd["_disc_logits.weight"], w)
        out["disc_loss"] = d["disc_loss"]
        out["loss"] = out["loss"] + disc_coef * d["disc_loss"]
    return out
