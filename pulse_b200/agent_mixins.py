"""Drop-in overrides for the reference's agent and task classes (method names, argument meaning and the keys of the
returned dictionaries are the reference's).  Mix them IN FRONT of the reference classes; rl_games keeps the training loop,
logging, checkpoint cadence and the experience buffer, Isaac Gym keeps the physics (INTEGRATION.md):

    from phc.learning.im_amp import IMAmpAgent
    class IMAmpAgentB200(AMPAgentB200Mixin, IMAmpAgent): pass
    runner.algo_factory.register_builder('im_amp', lambda **kw: IMAmpAgentB200(**kw))        # run_hydra.py:252-266

    from phc.env.tasks.humanoid_im_distill import HumanoidImDistill
    class HumanoidImDistillB200(HumanoidImDistillB200Mixin, HumanoidImB200Mixin, HumanoidImDistill): pass

These classes only route tensors to `PPOPolicy` / `PulseVAE` / `TeacherPNN` / `ReachTaskB200`; every number is computed by
the CUDA library (no CPU fallback).  rl_games and Isaac Gym are not installable here (SURVEY.md 8c): tests/test_gpu_boundary.py mixes
these classes in front of stand-in base classes (tests/standins.py) that carry the reference's attribute / method contract, and
tests/test_boundary_cpu.py checks that contract against names recorded from the unmodified reference sources
(tests/golden/contract_names.json).

Reference methods mirrored:
  CommonAgent.get_action_values   phc/learning/common_agent.py:262-288
  CommonAgent._eval_critic        :552-562
  CommonAgent.discount_values     :493-505   (+ _calc_advs :589-599 through `normalize_advantage`)
  AMPAgent.calc_gradients         phc/learning/amp_agent.py:605-760
  AMPAgent._optimize_kin          :771-849
  AMPAgent._calc_amp_rewards      :1011-1041
  AMPSeptBuilder.Network          phc/learning/amp_network_sept_builder.py (pulse_z_terrain.yaml's policy)  -> SeptPolicy
  HumanoidImDistill.step (teacher) phc/env/tasks/humanoid_im_distill.py:143-205
  HumanoidZ.compute_z_actions     phc/env/tasks/humanoid_z.py:81-155
  Humanoid._action_to_pd_targets  phc/env/tasks/humanoid.py:1392-1394
  HumanoidReach._update_task / _compute_task_obs / _compute_reward   phc/env/tasks/humanoid_reach.py:126-166
"""
from typing import Dict

import torch

from . import _lib
from .ppo import PPOPolicy
from .reach import ReachTaskB200
from .rollout import discount_values
from .sept import SeptPolicy
from .vae import PulseVAE, TeacherPNN, pd_targets


def _mlp_shape(seq) -> tuple:
    """(hidden units, activation name) of an nn.Sequential of Linear / activation modules (what network_builder._build_mlp makes)."""
    units = [int(m.out_features) for m in seq if hasattr(m, "out_features")]
    acts = [type(m).__name__.lower() for m in seq if not hasattr(m, "out_features")]
    act = "silu" if any(a == "silu" for a in acts) else "relu"
    return tuple(units), act


class AMPAgentB200Mixin:
    """Agent side.  Expects the reference agent's attributes (`vec_env`, `model`, `optimizer`, `horizon_length`, `normalize_value`, `e_clip`,
    `critic_coef`, `bounds_loss_coef`, `grad_norm`, `last_lr`, `_amp_minibatch_size`, `only_kin_loss`, `multi_gpu`, `running_mean_std`,
    `value_mean_std`, `_amp_input_mean_std`, ...).

    Ownership of state (so that rl_games' checkpoint cadence keeps working, common_agent.py:142-150):
      * network weights, Adam moments, observation / AMP-input normalisers: trained INSIDE the device library (`self._pulse`); every
        `get_weights / get_stats_weights / get_full_state_weights` first writes them back into `self.model`, `self.running_mean_std`,
        `self._amp_input_mean_std` and `self.optimizer.state`, so `save()` serialises what was trained;
      * value normaliser: `self.value_mean_std` stays the owner (the reference's `prepare_dataset` updates it, common_agent.py:372-374)
        and is mirrored into the library after every `prepare_dataset`;
      * `set_weights / set_stats_weights / set_full_state_weights` (restore) rebuild the device-side copy from the loaded modules."""

    def _pulse_policy(self):
        """Build the device-side networks lazily from the reference model's parameters (same checkpoint keys)."""
        if getattr(self, "_pulse", None) is None:
            task = self.vec_env.env.task
            dev = self.ppo_device
            net = self.model.a2c_network
            if getattr(task, "z_type", None) == "vae" and getattr(task, "distill", False):
                self._pulse = PulseVAE(self_obs_size=task.get_self_obs_size(), task_obs_size=task.get_task_obs_size(),
                                       num_actions=task.get_action_size(), latent=int(task.cfg["env"].get("embedding_size", 32)), device=dev,
                                       kin_lr=float(task.kin_lr), grad_norm=float(self.grad_norm), kld_coefficient=float(task.kld_coefficient),
                                       kld_coefficient_min=float(task.kld_coefficient_min), kld_anneal=bool(task.kld_anneal),
                                       ar1_coefficient=float(task.ar1_coefficient), use_ar1_prior=bool(task.use_ar1_prior),
                                       use_vae_prior_regu=bool(task.use_vae_prior_regu), horizon=int(self.horizon_length))
            elif hasattr(net, "_task_mlp"):                                             # amp_sept (pulse_z_terrain.yaml): shared task encoder
                detail = dict(task.get_task_obs_size_detail())
                if set(detail) != {"traj", "heightmap"}:
                    extra = sorted(set(detail) - {"traj", "heightmap"})
                    raise _lib.PulseError(f"the amp_sept policy covers the trajectory + height-map task observation only; task_obs_size_detail "
                                          f"has {extra or sorted(detail)} (the 'people' PointNet branch / 'heightmap_velocity' are not built)")
                units, act = _mlp_shape(net.actor_mlp)
                task_units, task_act = _mlp_shape(net._task_mlp)
                disc_units, _ = _mlp_shape(net._disc_mlp)
                self._pulse = SeptPolicy(self_obs_size=task.get_self_obs_size(), task_obs_size_detail=detail, task_units=task_units, units=units,
                                         act=act, task_act=task_act, num_actions=self.actions_num, with_disc=True, device=dev,
                                         lr=float(self.last_lr), e_clip=float(self.e_clip), critic_coef=float(self.critic_coef),
                                         bounds_coef=float(self.bounds_loss_coef), grad_norm=float(self.grad_norm),
                                         normalize_value=bool(self.normalize_value), amp_obs_size=int(self._amp_observation_space.shape[0]),
                                         disc_units=disc_units)
            else:
                units, act = _mlp_shape(net.actor_mlp)                                   # im.yaml / pulse_z_task.yaml / im_big.yaml alike
                disc_units, _ = _mlp_shape(net._disc_mlp)
                self._pulse = PPOPolicy(obs_size=self.obs_shape[0], num_actions=self.actions_num, units=units, act=act, device=dev,
                                        lr=float(self.last_lr), e_clip=float(self.e_clip), critic_coef=float(self.critic_coef),
                                        bounds_coef=float(self.bounds_loss_coef), grad_norm=float(self.grad_norm),
                                        normalize_value=bool(self.normalize_value), with_disc=True,
                                        amp_obs_size=int(self._amp_observation_space.shape[0]), disc_units=disc_units)
            self._pulse_load_from_model()
        return self._pulse

    # ------------------------------------------------------------------ state exchange with the reference objects
    def _pulse_stats_modules(self):
        return (("running_mean_std", getattr(self, "running_mean_std", None)), ("reward_mean_std", getattr(self, "value_mean_std", None)),
                ("amp_input_mean_std", getattr(self, "_amp_input_mean_std", None)))

    def _pulse_load_from_model(self) -> None:
        pol = self._pulse
        sd = {k: v.detach() for k, v in self.model.state_dict().items()}
        for sec, mod in self._pulse_stats_modules():
            if mod is not None:
                for k, v in mod.state_dict().items():
                    sd[f"{sec}.{k}"] = v.detach()
        pol.load_state_dict(sd)
        if isinstance(pol, PPOPolicy) and getattr(self, "optimizer", None) is not None:
            named = dict(self.model.named_parameters())
            state = {n: self.optimizer.state[p] for n, p in named.items() if p in self.optimizer.state and len(self.optimizer.state[p])}
            pol.load_optimizer_state(state)

    def _pulse_write_back(self) -> None:
        """Device-side training state -> the reference objects rl_games serialises."""
        pol = getattr(self, "_pulse", None)
        if pol is None:
            return
        sd = pol.state_dict()
        own = self.model.state_dict()
        with torch.no_grad():
            for k, v in sd.items():
                if k in own:
                    own[k].copy_(v.to(own[k].device, own[k].dtype))
            for sec, mod in self._pulse_stats_modules():
                if mod is None or (sec == "reward_mean_std" and isinstance(pol, PPOPolicy)):
                    continue                             # the value normaliser is owned by the reference module (see class docstring)
                st = mod.state_dict()
                for k in ("running_mean", "running_var", "count"):
                    if f"{sec}.{k}" in sd and k in st:
                        st[k].copy_(sd[f"{sec}.{k}"].to(st[k].device, st[k].dtype).reshape(st[k].shape))
            if isinstance(pol, PPOPolicy) and getattr(self, "optimizer", None) is not None:
                opt_state = pol.optimizer_state(gather=False)   # this may run on rank 0 only (rl_games saves there): train_epoch gathered
                for n, p in self.model.named_parameters():
                    if n in opt_state:
                        tgt = self.optimizer.state[p]
                        for k, v in opt_state[n].items():
                            tgt[k] = v.to(p.device) if k != "step" else v.to("cpu")

    def _pulse_mirror_value_stats(self) -> None:
        pol, mod = getattr(self, "_pulse", None), getattr(self, "value_mean_std", None)
        if pol is None or mod is None or getattr(pol, "value_rms", None) is None:
            return
        st = mod.state_dict()
        pol.value_rms.running_mean.copy_(st["running_mean"].double().reshape(-1))
        pol.value_rms.running_var.copy_(st["running_var"].double().reshape(-1))
        pol.value_rms.count.copy_(st["count"].double().reshape(()))
        pol.value_rms._refresh()

    def get_stats_weights(self):
        self._pulse_write_back()
        return super().get_stats_weights()

    def get_weights(self):
        self._pulse_write_back()
        return super().get_weights()

    def get_full_state_weights(self):
        self._pulse_write_back()
        return super().get_full_state_weights()

    def set_stats_weights(self, weights):
        super().set_stats_weights(weights)
        self._pulse = None                               # rebuilt from the restored modules at the next use

    def set_weights(self, weights):
        super().set_weights(weights)
        self._pulse = None

    def set_full_state_weights(self, weights):
        super().set_full_state_weights(weights)
        self._pulse = None

    def prepare_dataset(self, batch_dict):
        out = super().prepare_dataset(batch_dict)        # normalises values / returns and merges them into value_mean_std (common_agent.py:372-374)
        self._pulse_mirror_value_stats()
        return out

    def train_epoch(self):
        info = super().train_epoch()
        if getattr(self, "multi_gpu", False) and torch.distributed.is_initialized():   # hvd.sync_stats (common_agent.py:126-127)
            pol = self._pulse_policy()
            if isinstance(pol, PPOPolicy):
                pol.sync_stats(torch.distributed.get_world_size())
                pol.flat.gather_moments()     # peer-memory optimizer: the Adam moments are sharded; every rank re-assembles them here (once
                                              # per epoch, two all-reduces) so that a rank-0-only checkpoint write needs no collective
        return info

    # ------------------------------------------------------------------ rollout side
    def get_action_values(self, obs):
        pol = self._pulse_policy()
        res = pol.act(obs["obs"])
        # PulseVAE.act (only_kin_loss): the env is stepped with `mus` (amp_agent.py:244-246, :367-369); no PPO statistics are used,
        # so `actions` = `mus` and `neglogpacs` = 0 stand in for the sampled action and its likelihood
        out = {"actions": res.get("actions", res["mus"]), "mus": res["mus"], "sigmas": res["sigmas"], "values": res["values"],
               "neglogpacs": res.get("neglogpacs", torch.zeros(res["mus"].shape[0], device=res["mus"].device)), "rnn_states": None}
        return out

    def _eval_critic(self, obs_dict):
        pol = self._pulse_policy()
        if isinstance(pol, PulseVAE):
            return pol.value_rms.unnormalize(pol.eval_critic(obs_dict["obs"]))
        return pol.critic_values(obs_dict["obs"])

    def _calc_amp_rewards(self, amp_obs):
        pol = self._pulse_policy()
        if not hasattr(pol, "disc") or pol.disc is None:
            # distillation (only_kin_loss): the AMP reward is logged but does not enter the kin loss; the reference path keeps it
            return super()._calc_amp_rewards(amp_obs)
        return {"disc_rewards": pol.disc.rewards(amp_obs.reshape(-1, amp_obs.shape[-1])).reshape(*amp_obs.shape[:-1], 1)}

    def discount_values(self, mb_fdones, mb_values, mb_rewards, mb_next_values):
        """Returns the advantages in the reference's [T, N, 1] layout (the fused kernel produces them env-major)."""
        T, N = mb_fdones.shape[0], mb_fdones.shape[1]
        adv, _ = discount_values(mb_fdones, mb_values, mb_rewards, mb_next_values, gamma=float(self.gamma), tau=float(self.tau))
        return adv.view(N, T).t().unsqueeze(-1).contiguous()

    # ------------------------------------------------------------------ update side
    def calc_gradients(self, input_dict):
        pol = self._pulse_policy()
        world = 1
        if getattr(self, "multi_gpu", False) and torch.distributed.is_initialized():
            world = torch.distributed.get_world_size()
        self.train_result = {}
        if getattr(self, "only_kin_loss", False):
            self.train_result.update(self._optimize_kin({"obs_orig": input_dict["obs"], "kin_dict": input_dict["kin_dict"]}))
            zero = torch.tensor(0).float()
            self.train_result.update({"entropy": zero, "kl": zero, "last_lr": self.last_lr, "lr_mul": zero})
            return
        n = self._amp_minibatch_size
        M = input_dict["obs"].shape[0]
        pol.lr = float(self.last_lr)
        pol.reset_stats()                                    # per-minibatch statistics, as the reference logs them
        stats = pol.train_minibatch(input_dict["obs"], input_dict["actions"], input_dict["old_logp_actions"], input_dict["advantages"],
                                    input_dict["returns"], old_mu=input_dict["mu"], world_size=world,
                                    amp=(input_dict["amp_obs"][0:n], input_dict["amp_obs_replay"][0:n], input_dict["amp_obs_demo"][0:n]))
        s = stats / M                                        # fp64 on the device; .item() only where the reference logs
        self.train_result.update({"actor_loss": s[0], "critic_loss": s[1], "b_loss": s[2], "kl": s[3], "actor_clip_frac": s[4],
                                  "entropy": torch.zeros((), device=stats.device), "last_lr": self.last_lr, "lr_mul": 1.0})
        self.train_result.update(pol.disc.loss_tensors(n))   # disc_loss, disc_agent_acc, ... (AMPAgent._assemble_train_info reads them)

    def _optimize_kin(self, batch_dict):
        """batch_dict['obs_orig']: raw observations of the minibatch (normalised inside, as `_preproc_obs` does);
        batch_dict['kin_dict']: the flat [gt_action | progress_buf] rows assembled by `_assamble_kin_dict`."""
        pol = self._pulse_policy()
        kin = self._assamble_kin_dict(batch_dict["kin_dict"])
        M = kin["gt_action"].shape[0]
        world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
        pol.optimize_kin(batch_dict["obs_orig"], kin["gt_action"].contiguous(), kin["progress_buf"].reshape(-1).long().contiguous(),
                         update_obs_rms=not getattr(self, "temp_running_mean", False), world_size=world)
        info: Dict[str, object] = dict(pol.losses(M))
        info["kin_kld_w"] = pol.anneal(int(self.epoch_num))
        self.vec_env.env.task.kld_coefficient = pol.kld_coefficient
        return info


class PdTargetsB200Mixin:
    """Humanoid._action_to_pd_targets (humanoid.py:1392-1394) on the device library."""

    def _action_to_pd_targets(self, action):
        return pd_targets(action.contiguous(), self._pd_action_offset, self._pd_action_scale)


class HumanoidImDistillB200Mixin(PdTargetsB200Mixin):
    """HumanoidImDistill.step (humanoid_im_distill.py:143-205): the frozen teacher's action for the CURRENT observation goes
    into `kin_dict['gt_action']` before the env steps.  Covers the default distillation config (PNN + composer teacher,
    `env_im_vae.yaml:56-61`, same observation settings for teacher and student)."""

    def _pulse_teacher(self):
        if getattr(self, "_pulse_teacher_obj", None) is None:
            if not getattr(self, "has_pnn_distill", False) or getattr(self, "distill_z_model", False):
                raise _lib.PulseError("HumanoidImDistillB200Mixin covers the PNN + composer teacher only")
            pnn_sd = {k: v for k, v in self.pnn.state_dict().items()}
            comp_sd = {k: v for k, v in self.composer.state_dict().items()}
            units = [self.pnn.actors[0][i].out_features for i in range(0, len(self.pnn.actors[0]) - 1, 2)]
            cunits = [m.out_features for m in self.composer if hasattr(m, "out_features")][:-1]
            t = TeacherPNN(obs_size=self.get_obs_size(), num_actions=self.get_action_size(), prim_units=units, composer_units=cunits,
                           num_prim=int(self.num_prim_distill), composer_act=str(self.z_activation), device=self.device)
            t.load_weights(pnn_sd, comp_sd, self.running_mean, self.running_var)
            self._pulse_teacher_obj = t
        return self._pulse_teacher_obj

    def step(self, actions):
        from .flags_compat import flags_test
        if not flags_test() and self.save_kin_info:
            self.kin_dict["gt_action"] = self._pulse_teacher().gt_action(self.obs_buf).clone()
            self.kin_dict["progress_buf"] = self.progress_buf.clone()
        # the rest of Humanoid.step: pre_physics_step -> physics -> post_physics_step (base_task / humanoid.py)
        self.pre_physics_step(actions)
        self._physics_step()
        if self.device == "cpu":
            self.gym.fetch_results(self.sim, True)
        self.post_physics_step()


class HumanoidZB200Mixin(PdTargetsB200Mixin):
    """HumanoidZ.compute_z_actions (humanoid_z.py:81-155) for the 'vae' latent with the learned prior: the frozen prior and
    decoder of the distilled checkpoint on the tensor cores."""

    def _pulse_decoder(self):
        if getattr(self, "_pulse_vae", None) is None:
            if self.distill_z_type != "vae" or not self.use_vae_prior or self.z_all:
                raise _lib.PulseError("HumanoidZB200Mixin covers z_type 'vae' with use_vae_prior (pulse_z_task.yaml) only")
            ck = self._pulse_checkpoint            # the torch_ext.load_checkpoint(...) dict of models_path[0], kept by initialize_z_models
            vae = PulseVAE(self_obs_size=self.get_self_obs_size(), task_obs_size=ck["model"]["a2c_network.z_mlp.0.weight"].shape[1] - self.get_self_obs_size(),
                           num_actions=ck["model"]["a2c_network.mu.bias"].shape[0], latent=int(self.cfg["env"].get("embedding_size", 32)),
                           device=self.device, with_critic=False)
            vae.load_state_dict(dict(ck["model"], **{"running_mean_std.running_mean": ck["running_mean_std"]["running_mean"],
                                                     "running_mean_std.running_var": ck["running_mean_std"]["running_var"]}))
            self._pulse_vae = vae
        return self._pulse_vae

    def compute_z_actions(self, action_z):
        return self._pulse_decoder().compute_z_actions(self.obs_buf, action_z.contiguous())


class HumanoidReachB200Mixin:
    """HumanoidReach post-physics path (humanoid_reach.py:126-166, :224-250) in one launch: the first of `_compute_reward` /
    `_compute_reset` / `_compute_observations` after a physics step runs the fused kernel, the others return."""

    def _pulse_reach(self):
        if getattr(self, "_pulse_reach_obj", None) is None:
            names = self._body_names if hasattr(self, "_body_names") else None
            contact = [names[i] for i in self._contact_body_ids.tolist()] if names is not None else ("R_Ankle", "L_Ankle", "R_Toe", "L_Toe")
            r = ReachTaskB200(self.num_envs, device=self.device, reach_body_name=self.cfg["env"]["reachBodyName"], contact_bodies=contact,
                              tar_change_steps_min=self._tar_change_steps_min, tar_change_steps_max=self._tar_change_steps_max,
                              tar_dist_max=self._tar_dist_max, tar_height_min=self._tar_height_min, tar_height_max=self._tar_height_max,
                              max_episode_length=int(self.max_episode_length), enable_early_termination=bool(self._enable_early_termination))
            r.termination_heights.copy_(self._termination_heights.reshape(-1)[:24])
            # share the reference's buffers so every other method of the task keeps seeing them
            r._tar_pos, r._tar_change_steps = self._tar_pos, self._tar_change_steps
            r.obs_buf, r.rew_buf, r.reset_buf, r._terminate_buf = self.obs_buf, self.rew_buf, self.reset_buf, self._terminate_buf
            self._pulse_reach_obj, self._pulse_reach_pending = r, False
        return self._pulse_reach_obj

    def _update_task(self):
        self._pulse_reach().update_task(self.progress_buf)

    def _pulse_fused(self):
        self._pulse_reach().post_physics_step(self._rigid_body_state_reshaped, self.progress_buf, self._contact_forces)
        self._pulse_reach_pending = True

    def _compute_reward(self, actions):
        self._pulse_fused()

    def _compute_reset(self):
        if not getattr(self, "_pulse_reach_pending", False):
            self._pulse_fused()

    def _compute_observations(self, env_ids=None):
        if env_ids is None and getattr(self, "_pulse_reach_pending", False):
            self._pulse_reach_pending = False
            return
        self._pulse_reach_pending = False
        if env_ids is None:
            self._pulse_fused()
            self._pulse_reach_pending = False
        else:
            super()._compute_observations(env_ids)   # reset-time subset: the reference path (rare, variable size)
