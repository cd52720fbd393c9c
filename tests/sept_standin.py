"""Stand-in for the reference agent that trains pulse_z_terrain.yaml's `amp_sept` network (rl_games and Isaac Gym are not installable
here): the attributes and methods AMPAgentB200Mixin reads, with `model.a2c_network` an nn.Module that carries the reference network's
parameter names and whose arithmetic is oracle/sept_oracle.py."""
import types

import torch
import torch.nn as nn

from tests.sept_fixture import normalise


class _Rms(nn.Module):
    def __init__(self, mean, var):
        super().__init__()
        self.register_buffer("running_mean", mean.double().clone())
        self.register_buffer("running_var", var.double().clone())
        self.register_buffer("count", torch.ones((), dtype=torch.float64))


def _seq(n_in, units, act):
    mods = []
    for u in units:
        mods += [nn.Linear(n_in, u), act()]
        n_in = u
    return nn.Sequential(*mods)


class SeptNetwork(nn.Module):
    """AMPSeptBuilder.Network's parameters (names and shapes); eval_actor / eval_critic are the oracle's."""

    def __init__(self, d):
        super().__init__()
        S, T, E = d["S"], d["traj"] + d["heightmap"], d["task_units"][-1]
        self.self_obs_size = S
        self._task_mlp = _seq(T, d["task_units"], nn.SiLU)
        self.actor_mlp, self.critic_mlp = _seq(S + E, d["units"], nn.SiLU), _seq(S + E, d["units"], nn.SiLU)
        self.mu, self.value = nn.Linear(d["units"][-1], d["A"]), nn.Linear(d["units"][-1], 1)
        self.sigma = nn.Parameter(torch.full((d["A"],), -1.0), requires_grad=False)
        self._disc_mlp = _seq(d["amp"], d["disc_units"], nn.ReLU)
        self._disc_logits = nn.Linear(d["disc_units"][-1], 1)

    def eval_actor(self, obs):
        from oracle import sept_oracle as so
        return so.eval_actor(dict(self.named_parameters()), obs, self.self_obs_size)

    def eval_critic(self, obs):
        from oracle import sept_oracle as so
        return so.eval_critic(dict(self.named_parameters()), obs, self.self_obs_size)


class SeptAgentStandin:
    def __init__(self, d, sd, batch, device, detail=None):
        net = SeptNetwork(d).to(device)
        net.load_state_dict({k: v.to(device) for k, v in sd.items()})
        self.model = nn.Module()
        self.model.a2c_network = net
        detail = detail or {"traj": d["traj"], "heightmap": d["heightmap"]}
        task = types.SimpleNamespace(get_self_obs_size=lambda: d["S"], get_task_obs_size_detail=lambda: dict(detail))
        self.vec_env = types.SimpleNamespace(env=types.SimpleNamespace(task=task))
        self.ppo_device = device
        self.optimizer = torch.optim.Adam(self.model.parameters(), lr=2e-5)
        self.obs_shape, self.actions_num = (d["S"] + d["traj"] + d["heightmap"],), d["A"]
        self.last_lr, self.e_clip, self.critic_coef, self.bounds_loss_coef, self.grad_norm = 2e-5, 0.2, 5.0, 10.0, 50.0
        self.normalize_value, self.multi_gpu, self.only_kin_loss = True, False, False
        self._amp_observation_space = types.SimpleNamespace(shape=(d["amp"],))
        self._amp_minibatch_size = d["B"]
        self.running_mean_std = _Rms(batch["obs_mean"], batch["obs_var"]).to(device)
        self.value_mean_std = _Rms(torch.zeros(1), torch.ones(1)).to(device)
        self._amp_input_mean_std = _Rms(batch["amp_mean"], batch["amp_var"]).to(device)

    def reference_outputs(self, obs):
        """(mu, value) of the reference network on raw observations (eval-mode normaliser; the value normaliser is at its identity)."""
        rms = self.running_mean_std
        x = normalise(obs, rms.running_mean.float(), rms.running_var.float())
        return self.model.a2c_network.eval_actor(x), self.model.a2c_network.eval_critic(x)

    # rl_games' checkpoint hooks (the mixin writes its state back before delegating here)
    def get_weights(self):
        return self.model.state_dict()

    def set_weights(self, weights):
        if weights is not None:
            self.model.load_state_dict(weights)
