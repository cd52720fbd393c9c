"""Stand-in base classes for the boundary tests (TEST INFRASTRUCTURE).

Isaac Gym and rl_games are not installable (SURVEY.md 8c), so `HumanoidImB200Mixin` / `AMPAgentB200Mixin` cannot be mixed in front of
the real `phc.env.tasks.humanoid_im.HumanoidIm` / `phc.learning.im_amp.IMAmpAgent` here.  These classes carry exactly the part of the
reference's attribute / method contract the mixins touch -- names, shapes, dtypes and call order as in the cited reference lines -- and
nothing else.  tests/test_boundary_cpu.py checks that every name used here occurs in the unmodified reference sources it is cited from,
against the pairs recorded from those sources (tests/golden/contract_names.json, make_golden_contract.py).
"""
import types

import torch

CONTRACT = {
    # attribute / method names of the reference TASK the mixin reads or overrides -> reference file that defines them
    "task": {
        "phc/env/tasks/humanoid_im.py": ["_compute_reward", "_compute_reset", "_compute_observations", "_sampled_motion_ids", "_motion_start_times",
                                         "_motion_start_times_offset", "_global_offset", "_cycle_counter", "reward_specs", "power_reward",
                                         "power_coefficient", "_reset_bodies_id", "_termination_distances", "ref_body_pos", "ref_body_vel",
                                         "ref_body_rot", "ref_dof_pos", "reward_raw", "obs_v", "_fut_tracks", "zero_out_far", "_occl_training",
                                         "_full_body_reward", "_track_bodies_id", "cycle_motion", "resample_motions", "_sample_time", "_compute_task_obs",
                                         "_num_traj_samples", "_traj_sample_timestep", "_fut_tracks_dropout", "ref_body_pos_subset"],
        "phc/env/tasks/humanoid.py": ["_rigid_body_state_reshaped", "_dof_vel", "_dof_pos", "dof_force_tensor", "progress_buf", "obs_buf",
                                      "self_obs_buf", "rew_buf", "reset_buf", "_terminate_buf", "max_episode_length", "_enable_early_termination",
                                      "self_obs_v", "_humanoid_root_states", "post_physics_step", "_has_dof_subset", "_reset_envs",
                                      "_reset_env_tensors", "_rigid_body_pos", "_rigid_body_rot", "_rigid_body_vel", "_rigid_body_ang_vel",
                                      "_contact_forces", "_humanoid_actor_ids", "_has_upright_start"],
        "phc/env/tasks/humanoid_amp.py": ["_update_hist_amp_obs", "_compute_amp_observations", "_amp_obs_buf", "_num_amp_obs_steps", "_motion_lib",
                                          "amp_obs_v", "_state_init", "_reset_default_env_ids", "_reset_ref_env_ids", "_reset_ref_motion_ids",
                                          "_reset_ref_motion_times", "_state_reset_happened", "_reset_rb_pos", "_reset_rb_rot", "_reset_rb_vel",
                                          "_reset_rb_ang_vel", "_refresh_sim_tensors"],
        "phc/env/tasks/humanoid_im_getup.py": ["_recovery_counter"],
    },
    # names of the reference AGENT the mixin reads, overrides or calls through super()
    "agent": {
        "phc/learning/amp_agent.py": ["calc_gradients", "_optimize_kin", "_calc_amp_rewards", "get_stats_weights", "set_stats_weights",
                                      "get_full_state_weights", "set_full_state_weights", "prepare_dataset", "train_epoch", "_amp_input_mean_std",
                                      "value_mean_std", "_amp_minibatch_size", "_amp_observation_space", "only_kin_loss", "_assamble_kin_dict",
                                      "temp_running_mean", "train_result"],
        "phc/learning/common_agent.py": ["get_action_values", "_eval_critic", "discount_values", "bounds_loss_coef", "running_mean_std", "last_lr",
                                         "e_clip", "critic_coef", "grad_norm", "normalize_value", "horizon_length", "multi_gpu", "ppo_device",
                                         "gamma", "tau", "epoch_num"],
    },
}


class RunningMeanStdModule(torch.nn.Module):
    """phc/utils/running_mean_std.py:9-109 (the nn.Module rl_games checkpoints: buffers running_mean / running_var / count, fp64)."""

    def __init__(self, size, epsilon=1e-5):
        super().__init__()
        self.epsilon = epsilon
        self.register_buffer("running_mean", torch.zeros(size, dtype=torch.float64))
        self.register_buffer("running_var", torch.ones(size, dtype=torch.float64))
        self.register_buffer("count", torch.ones((), dtype=torch.float64))

    def forward(self, x, unnorm=False):
        mean, var = self.running_mean.float(), self.running_var.float()
        if unnorm:
            return torch.sqrt(var + self.epsilon) * torch.clamp(x, -5.0, 5.0) + mean
        y = torch.clamp((x - mean) / torch.sqrt(var + self.epsilon), -5.0, 5.0)
        if self.training:   # update AFTER normalising (:96-107)
            n = x.shape[0]
            bm, bv = x.double().mean(0), x.double().var(0)
            delta = bm - self.running_mean
            tot = self.count + n
            m2 = self.running_var * self.count + bv * n + delta ** 2 * self.count * n / tot
            self.running_mean.copy_(self.running_mean + delta * n / tot)
            self.running_var.copy_(m2 / tot)
            self.count.copy_(tot)
        return y


def mlp(sizes, act=torch.nn.ReLU):
    layers = []
    for i in range(len(sizes) - 1):
        layers += [torch.nn.Linear(sizes[i], sizes[i + 1]), act()]
    return torch.nn.Sequential(*layers)


class AMPNetwork(torch.nn.Module):
    """Parameter names of `AMPBuilder.Network` (amp_network_builder.py:20-249, network_builder.py:190-291): actor_mlp / critic_mlp /
    mu / value / sigma / _disc_mlp / _disc_logits, wrapped as `a2c_network` by ModelAMPContinuous (amp_models.py:23-60)."""

    def __init__(self, obs=934, actions=69, units=(1024, 512), amp=1960, disc_units=(1024, 512)):
        super().__init__()
        self.actor_mlp, self.critic_mlp = mlp((obs,) + tuple(units)), mlp((obs,) + tuple(units))
        self.mu, self.value = torch.nn.Linear(units[-1], actions), torch.nn.Linear(units[-1], 1)
        self.sigma = torch.nn.Parameter(torch.full((actions,), -2.9), requires_grad=False)
        self._disc_mlp = mlp((amp,) + tuple(disc_units))
        self._disc_logits = torch.nn.Linear(disc_units[-1], 1)


class AMPModel(torch.nn.Module):
    def __init__(self, **kw):
        super().__init__()
        self.a2c_network = AMPNetwork(**kw)


class StandInAMPAgent:
    """The rl_games A2CBase / CommonAgent / AMPAgent surface `AMPAgentB200Mixin` builds on."""

    def __init__(self, task, device, seed=0, **net_kw):
        torch.manual_seed(seed)
        self.vec_env = types.SimpleNamespace(env=types.SimpleNamespace(task=task))
        self.ppo_device = self.device = device
        self.model = AMPModel(**net_kw).to(device)
        self.last_lr, self.e_clip, self.critic_coef, self.bounds_loss_coef, self.grad_norm = 2e-5, 0.2, 5.0, 10.0, 50.0   # im.yaml:55-75
        self.optimizer = torch.optim.Adam(self.model.parameters(), float(self.last_lr), eps=1e-8, weight_decay=0.0)        # common_agent.py:67
        self.obs_shape, self.actions_num = (self.model.a2c_network.actor_mlp[0].in_features,), self.model.a2c_network.mu.out_features
        self.normalize_input = self.normalize_value = self._normalize_amp_input = True
        amp = self.model.a2c_network._disc_mlp[0].in_features
        self._amp_observation_space = types.SimpleNamespace(shape=(amp,))
        self.running_mean_std = RunningMeanStdModule(self.obs_shape[0]).to(device)
        self.value_mean_std = RunningMeanStdModule(1).to(device)               # amp_agent.py:47-48
        self._amp_input_mean_std = RunningMeanStdModule(amp).to(device)        # amp_agent.py:50-51
        self._amp_minibatch_size, self.horizon_length, self.gamma, self.tau = 4096, 32, 0.99, 0.95
        self.multi_gpu, self.only_kin_loss, self.epoch_num, self.frame = False, False, 0, 0
        self.dataset_dict = None

    # ---- A2CBase [rl_games, 3P-memory] + AMPAgent (amp_agent.py:81-119, :181-189) ----
    def get_stats_weights(self):
        return {"running_mean_std": self.running_mean_std.state_dict(), "reward_mean_std": self.value_mean_std.state_dict(),
                "amp_input_mean_std": self._amp_input_mean_std.state_dict()}

    def get_weights(self):
        state = self.get_stats_weights()
        state["model"] = self.model.state_dict()
        return state

    def get_full_state_weights(self):
        state = self.get_weights()
        state.update(epoch=self.epoch_num, optimizer=self.optimizer.state_dict(), frame=self.frame)
        return state

    def set_stats_weights(self, weights):
        self.running_mean_std.load_state_dict(weights["running_mean_std"])
        self.value_mean_std.load_state_dict(weights["reward_mean_std"])
        self._amp_input_mean_std.load_state_dict(weights["amp_input_mean_std"])

    def set_weights(self, weights):
        self.model.load_state_dict(weights["model"])
        self.set_stats_weights(weights)

    def set_full_state_weights(self, weights):
        self.set_weights(weights)
        self.epoch_num, self.frame = weights["epoch"], weights.get("frame", 0)
        self.optimizer.load_state_dict(weights["optimizer"])

    # ---- CommonAgent.prepare_dataset (common_agent.py:357-398): values / returns through value_mean_std in TRAIN mode ----
    def prepare_dataset(self, batch_dict):
        self.value_mean_std.train()
        values = self.value_mean_std(batch_dict["values"])
        returns = self.value_mean_std(batch_dict["returns"])
        self.value_mean_std.eval()
        self.dataset_dict = dict(batch_dict, old_values=values, returns=returns)
        return self.dataset_dict

    def train_epoch(self):
        return {}

    def _calc_amp_rewards(self, amp_obs):
        raise AssertionError("the mixin must serve the AMP reward from the device library")


class StandInHumanoidIm:
    """The Humanoid / HumanoidAMP / HumanoidIm surface `HumanoidImB200Mixin` builds on: Isaac-Gym shaped state views, the task buffers of
    `HumanoidIm.__init__` (humanoid_im.py:36-110) and `Humanoid.post_physics_step`'s call order (humanoid.py:1315-1346,
    humanoid_amp.py:194-210)."""

    def __init__(self, motion_lib, z, device, getup=False):
        n = z["body_state"].shape[0]
        dev = torch.device(device)
        self.device, self.num_envs = dev, n
        self._motion_lib = motion_lib
        self.dt = float(torch.tensor(1.0 / 60.0, dtype=torch.float32) * 2)
        self.reward_specs = {"k_pos": 100, "k_rot": 10, "k_vel": 0.1, "k_ang_vel": 0.1, "w_pos": 0.5, "w_rot": 0.3, "w_vel": 0.1, "w_ang_vel": 0.1}
        self.power_reward, self.power_coefficient = True, 0.0005
        self._reset_bodies_id = torch.tensor([j for j in range(24) if j not in (3, 4, 7, 8)], device=dev)
        self._track_bodies_id = torch.arange(24, device=dev)
        self._termination_distances = torch.full((1, 24), 0.25, device=dev)
        self._enable_early_termination, self.cycle_motion, self.max_episode_length = True, False, 300
        self.obs_v, self.self_obs_v, self.amp_obs_v = 6, 1, 1
        self._fut_tracks = self.zero_out_far = self._occl_training = self.add_obs_noise = False
        self._full_body_reward, self._has_dof_subset, self._num_amp_obs_steps = True, True, 10
        # simulator tensors (gymtorch views): 26 bodies, 72 dofs x (pos, vel), 2 actors
        self._rigid_body_state_reshaped = torch.zeros(n, 26, 13, device=dev)
        self._rigid_body_state_reshaped[:, :24] = z["body_state"].to(dev)
        self._dof_state = torch.zeros(n, 72, 2, device=dev)
        self._dof_state[:, :69, 0], self._dof_state[:, :69, 1] = z["dof_pos"].to(dev), z["dof_vel"].to(dev)
        self._dof_pos, self._dof_vel = self._dof_state[:, :69, 0], self._dof_state[:, :69, 1]
        self.dof_force_tensor = z["dof_force"].to(dev)
        self._root_states = torch.zeros(n, 2, 13, device=dev)
        self._humanoid_root_states = self._root_states[:, 0]
        # task buffers
        self.progress_buf = z["progress_buf"].to(dev).clone() - 1            # post_physics_step increments first
        self._sampled_motion_ids = z["motion_ids"].to(dev)
        self._motion_start_times, self._motion_start_times_offset = z["start_times"].to(dev), z["start_offset"].to(dev)
        self._global_offset, self._cycle_counter = z["global_offset"].to(dev), z["cycle_counter"].to(dev)
        self.obs_buf, self.self_obs_buf = torch.zeros(n, 934, device=dev), torch.zeros(n, 358, device=dev)
        self.rew_buf, self.reward_raw = torch.zeros(n, device=dev), torch.zeros(n, 5, device=dev)
        self.reset_buf, self._terminate_buf = torch.ones(n, dtype=torch.long, device=dev), torch.ones(n, dtype=torch.long, device=dev)
        self.ref_body_pos, self.ref_body_vel = torch.zeros(n, 24, 3, device=dev), torch.zeros(n, 24, 3, device=dev)
        self.ref_body_rot, self.ref_dof_pos = torch.zeros(n, 24, 4, device=dev), torch.zeros(n, 69, device=dev)
        self._amp_obs_buf = torch.zeros(n, 10, 196, device=dev)
        self._curr_amp_obs_buf, self._hist_amp_obs_buf = self._amp_obs_buf[:, 0], self._amp_obs_buf[:, 1:]   # humanoid_amp.py:123-124
        if getup:
            self._recovery_counter = torch.zeros(n, device=dev, dtype=torch.int)     # humanoid_im_getup.py:61
        self.extras, self.actions = {}, None
        # reset side (humanoid.py:196-243, humanoid_amp.py:95-110)
        rb = self._rigid_body_state_reshaped[:, :24]
        self._rigid_body_pos, self._rigid_body_rot = rb[..., 0:3], rb[..., 3:7]
        self._rigid_body_vel, self._rigid_body_ang_vel = rb[..., 7:10], rb[..., 10:13]
        self._contact_forces = torch.ones(n, 26, 3, device=dev)
        self._humanoid_actor_ids = (2 * torch.arange(n, device=dev)).to(torch.int32)         # 2 actors per env
        self._state_init = types.SimpleNamespace(name="Random")                              # HumanoidAMP.StateInit.Random
        self._state_reset_happened = False
        self._reset_default_env_ids, self._reset_ref_env_ids = [], []
        self.gym_calls = []
        self._sim_rigid_body_state = self._rigid_body_state_reshaped.clone()                 # what gym's refresh writes back

    def post_physics_step(self):
        self.progress_buf += 1                       # humanoid.py:1317
        self._compute_reward(self.actions)
        self._compute_reset()
        self._compute_observations()
        self.extras["terminate"] = self._terminate_buf
        self._update_hist_amp_obs()                  # humanoid_amp.py:197-198
        self._compute_amp_observations()
        self.extras["amp_obs"] = self._amp_obs_buf.view(-1, 1960)

    # the reference implementations behind the mixin (only reached for configurations the mixin hands back)
    def _update_hist_amp_obs(self, env_ids=None):    # humanoid_amp.py:622-630
        if env_ids is None:
            self._hist_amp_obs_buf[:] = self._amp_obs_buf[:, 0:9].clone()
        else:
            self._hist_amp_obs_buf[env_ids] = self._amp_obs_buf[env_ids, 0:9]

    def _compute_amp_observations(self, env_ids=None):
        raise AssertionError("reference AMP path reached: the mixin should have served the default configuration")

    def resample_motions(self):
        pass

    def _reset_envs(self, env_ids):
        raise AssertionError("reference reset path reached: the mixin should have served StateInit.Random")

    def _reset_env_tensors(self, env_ids):           # humanoid.py:589-609 (the gym setters are recorded instead of executed)
        env_ids_int32 = self._humanoid_actor_ids[env_ids]
        self.gym_calls.append(("set_actor_root_state_tensor_indexed", env_ids_int32.clone(), len(env_ids_int32)))
        self.gym_calls.append(("set_dof_state_tensor_indexed", env_ids_int32.clone(), len(env_ids_int32)))
        self.progress_buf[env_ids] = 0
        self.reset_buf[env_ids] = 0
        self._terminate_buf[env_ids] = 0
        self._contact_forces[env_ids] = 0

    def _refresh_sim_tensors(self):                  # humanoid_amp.py:598-620
        self._rigid_body_state_reshaped.copy_(self._sim_rigid_body_state)      # gym.refresh_rigid_body_state_tensor: the simulator's (stale) bodies
        if self._state_reset_happened and "_reset_rb_pos" in self.__dict__:
            env_ids = self._reset_ref_env_ids
            if len(env_ids) > 0:
                self._rigid_body_pos[env_ids] = self._reset_rb_pos
                self._rigid_body_rot[env_ids] = self._reset_rb_rot
                self._rigid_body_vel[env_ids] = self._reset_rb_vel
                self._rigid_body_ang_vel[env_ids] = self._reset_rb_ang_vel
                self._state_reset_happened = False
