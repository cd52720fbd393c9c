"""PULSE VAE distillation on the GPU (SURVEY K17-K20): host-side mirror of

  AMPZBuilder.Network            phc/learning/amp_network_z_builder.py:24-557   -> PulseVAE (encoder / prior / decoder / critic stacks)
    eval_actor(return_extra)     :341-467, form_embedding :79-121               -> PulseVAE.eval_actor
    compute_prior                :226-241                                       -> PulseVAE.compute_prior
    eval_critic                  :249-339                                       -> PulseVAE.eval_critic
  AMPAgent._optimize_kin         phc/learning/amp_agent.py:771-849              -> PulseVAE.optimize_kin
  HumanoidImDistill.step         phc/env/tasks/humanoid_im_distill.py:143-205   -> TeacherPNN.gt_action  (frozen PNN + composer)
  HumanoidZ.compute_z_actions    phc/env/tasks/humanoid_z.py:81-155             -> PulseVAE.compute_z_actions
  Humanoid._action_to_pd_targets phc/env/tasks/humanoid.py:1222-1247,1392-1394  -> pd_targets

Every dense layer is a wgmma GEMM (`pulse_gemm_bf16`), forward and explicit backward; the row-wise pieces between them are
the kernels of csrc/vae_ops.cu.  Layout notes:
  * the decoder input is stored as [z (E) | self_obs (S) | 0-pad], i.e. the reference's `cat([self_obs, z])` with the two
    blocks swapped, so the latent window starts on a 16-byte boundary (its input gradient is one small GEMM on W0[:, :E]);
    layer-0 weight columns are permuted on checkpoint import / export (`MLP.in_perm`);
  * `z_mu` / `z_logvar` (and `z_prior_mu` / `z_prior_logvar`) are ONE fused [2E, K] head: columns [0,E) = mu, [E,2E) = logvar.
There is no CPU fallback: without libpulse_b200.so / a GPU every call raises.
"""
import ctypes as C
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .nets import MLP, FlatParams, pad8, pad_k
from .ppo import RunningMeanStdB200


def _split_heads(sd: Dict[str, torch.Tensor], mu_name: str, lv_name: str):
    return (torch.cat([sd[f"{mu_name}.weight"], sd[f"{lv_name}.weight"]], dim=0), torch.cat([sd[f"{mu_name}.bias"], sd[f"{lv_name}.bias"]], dim=0))


class PulseVAE:
    def __init__(self, self_obs_size: int = 358, task_obs_size: int = 576, num_actions: int = 69, latent: int = 32,
                 task_units: Sequence[int] = (1536, 1024, 512), dec_units: Sequence[int] = (3096, 2048, 1024), device="cuda:0", seed: int = 0,
                 kin_lr: float = 5e-4, grad_norm: float = 50.0, kld_coefficient: float = 0.01, kld_coefficient_min: float = 0.001,
                 kld_anneal: bool = True, ar1_coefficient: float = 0.005, use_ar1_prior: bool = True, use_vae_prior_regu: bool = False,
                 use_vae_clamped_prior: bool = True, vae_var_clamp_max: float = 2.0, horizon: int = 32, with_critic: bool = True,
                 logstd: float = -2.9):
        if latent > 128 or latent % 8 != 0:
            # embedding_size 32 for PULSE (env_im_vae.yaml), 48 for PULSE-X (env_pulsex_amp.yaml); the encoder's training kernels
            # (pulse_vae_reparam_philox, pulse_vae_latent_loss) serve up to 32 and refuse more, the frozen prior and decoder any size here
            raise _lib.PulseError("latent size must be a multiple of 8 and <= 128")
        if self_obs_size % 2 != 0:
            raise _lib.PulseError("self observation size must be even (pair-wise bf16 copies)")
        self.device = torch.device(device)
        self.S, self.Tk, self.A, self.E = self_obs_size, task_obs_size, num_actions, latent
        self.obs_size = self_obs_size + task_obs_size
        self.kin_lr, self.grad_norm, self.horizon = kin_lr, grad_norm, horizon
        self.kld_coefficient, self.kld_coefficient_min, self.kld_anneal = kld_coefficient, kld_coefficient_min, kld_anneal
        self.ar1_coefficient, self.use_ar1_prior, self.use_vae_prior_regu = ar1_coefficient, use_ar1_prior, use_vae_prior_regu
        self.clamp, self.clamp_lo, self.clamp_hi = use_vae_clamped_prior, -5.0, float(vae_var_clamp_max)
        E, S = latent, self_obs_size
        self.flat = FlatParams(self.device)          # what kin_optimizer updates (amp_agent.py:67): encoder, prior, decoder
        tu, du = list(task_units), list(dec_units)
        # z_mlp = [Linear+SiLU]*3 + Linear(512, 5E), then the fused z_mu | z_logvar head (:492-497, :510-512)
        self.enc = MLP(self.flat, self.obs_size, tu + [5 * E], 2 * E, "silu", hidden_acts=["silu"] * len(tu) + [None])
        self.prior = MLP(self.flat, S, tu, 2 * E, "silu")                                # z_prior + z_prior_mu | z_prior_logvar (:516-519)
        perm = torch.cat([torch.arange(S, S + E), torch.arange(0, S)])                   # internal [z | self] <- reference [self | z]
        self.dec = MLP(self.flat, S + E, du, num_actions, "silu", input_grad_cols=E, in_perm=perm)   # actor_mlp + mu
        self.flat.finalize()
        self.frozen = None
        self.critic_z = self.critic = None
        if with_critic:                              # evaluated in the rollout, never trained in only_kin_loss mode
            self.frozen = FlatParams(self.device)
            self.critic_z = MLP(self.frozen, self.obs_size, tu, E, "silu")               # critic_z_mlp (:557-)
            self.critic = MLP(self.frozen, S + E, du, 1, "silu", in_perm=perm)           # critic_mlp + value
            self.frozen.finalize(peer=False)      # never optimised: plain device memory
        gen = torch.Generator(device=self.device).manual_seed(seed)
        for m in (self.enc, self.prior, self.dec, self.critic_z, self.critic):
            if m is not None:
                m.init_default(gen)
                for l in m.layers:                   # the builder zero-initialises every bias (network_builder.py:281-284)
                    l.bias.zero_()
        self.logstd = torch.full((num_actions,), logstd, device=self.device)
        self.obs_rms = RunningMeanStdB200(self.obs_size, self.device)
        self.value_rms = RunningMeanStdB200(1, self.device)
        self.Kp = pad_k(self.obs_size)
        self.stats = torch.zeros(8, dtype=torch.float64, device=self.device)
        self.lib = _lib.load()
        self._bufs: Dict[tuple, dict] = {}
        self._side = None
        self.rng_seed = (int(seed) * 0x9E3779B97F4A7C15 + 0x452821E638D01377) & (2 ** 64 - 1)
        self.rng_offset = torch.zeros(1, dtype=torch.int64, device=self.device)    # uint64 counter read by pulse_vae_reparam_philox

    # ------------------------------------------------------------------ buffers
    def _buf(self, M: int) -> dict:
        if M not in self._bufs:
            dev, bf = self.device, torch.bfloat16
            E = self.E
            self._bufs[M] = {
                "x": torch.zeros(M, self.Kp, device=dev, dtype=bf),                          # normalised obs (encoder / critic_z input)
                "prior_in": torch.zeros(M, pad_k(self.S), device=dev, dtype=bf),             # normalised self obs
                "dec_in": torch.zeros(M, pad_k(self.S + E), device=dev, dtype=bf),           # [z | self obs | 0]
                "critic_in": torch.zeros(M, pad_k(self.S + E), device=dev, dtype=bf),        # [critic_z | self obs | 0]
                "noise": torch.zeros(M, E, device=dev),
                "dpred": torch.zeros(M, pad8(self.A), device=dev, dtype=bf),
                "d_enc": torch.zeros(M, 2 * E, device=dev, dtype=bf), "d_prior": torch.zeros(M, 2 * E, device=dev, dtype=bf),
            }
        return self._bufs[M]

    def _st(self):
        return _lib.current_stream(self.device)

    def _normalize_obs(self, obs: torch.Tensor, b: dict, update: bool = False) -> None:
        """rl_games `norm_obs` (RunningMeanStd, clamp +-5) into the encoder operand, then the self-observation columns into the
        prior operand and the decoder / critic input windows."""
        if update:
            self.obs_rms.normalize_update(obs, b["x"])
        else:
            self.obs_rms.normalize_into(obs, b["x"])
        E, S = self.E, self.S
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_copy_cols_bf16(b["x"].data_ptr(), b["x"].stride(0), obs.shape[0], S, b["prior_in"].data_ptr(),
                                                     b["prior_in"].stride(0), b["dec_in"][:, E:].data_ptr(), b["dec_in"].stride(0), self._st()),
                       "pulse_copy_cols_bf16")

    def _reparam(self, head: torch.Tensor, noise: Optional[torch.Tensor], mode: int, dst: torch.Tensor, rows: int, clamp: Optional[bool] = None):
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_vae_reparam(head.data_ptr(), head.stride(0), _lib.ptr(noise), noise.stride(0) if noise is not None else 0,
                                                  rows, self.E, mode, int(self.clamp if clamp is None else clamp), self.clamp_lo, self.clamp_hi,
                                                  dst.data_ptr(), dst.stride(0), None, 0, self._st()), "pulse_vae_reparam")

    # ------------------------------------------------------------------ forward pieces
    def eval_actor(self, obs: torch.Tensor, noise: Optional[torch.Tensor] = None, use_mean: bool = False, train: bool = False,
                   update_obs_rms: bool = False) -> Dict[str, torch.Tensor]:
        """eval_actor(return_extra=True): mu (the predicted action) and the posterior head.  `noise` injects the
        reparameterisation draw (the reference's "z_noise" path, :89-90); use_mean = flags.test (:94-95).
        Returned tensors are views of reused workspaces."""
        M = obs.shape[0]
        b = self._buf(M)
        self._normalize_obs(obs, b, update_obs_rms)
        head = self.enc.forward(b["x"], train=train)
        if noise is None and not use_mean:
            noise = b["noise"].normal_()
        self._reparam(head, noise, _lib.Z_MEAN if use_mean else _lib.Z_SAMPLE, b["dec_in"], M)
        mu = self.dec.forward(b["dec_in"], train=train)
        return {"mus": mu, "sigmas": torch.exp(self.logstd).expand(M, self.A), "enc_head": head, "noise": noise,
                "vae_mu": head[:, :self.E], "vae_log_var_raw": head[:, self.E:]}

    def compute_prior(self, obs: Optional[torch.Tensor] = None, train: bool = False, M: Optional[int] = None) -> torch.Tensor:
        """compute_prior: fp32 [M, 2E] = prior_mu | RAW prior log-variance (the clamp is applied by the consumers).
        obs None: reuse the operands of the preceding eval_actor call on M rows."""
        if obs is not None:
            M = obs.shape[0]
            self._normalize_obs(obs, self._buf(M))
        return self.prior.forward(self._buf(M)["prior_in"], train=train)

    def eval_critic(self, obs: Optional[torch.Tensor] = None, M: Optional[int] = None) -> torch.Tensor:
        """eval_critic, z_type 'vae' (:325-339): value = critic_mlp([self_obs, critic_z_mlp(obs)]) (normalised value)."""
        if self.critic is None:
            raise _lib.PulseError("PulseVAE was built without the critic stacks")
        if obs is not None:
            M = obs.shape[0]
            self._normalize_obs(obs, self._buf(M))
        b = self._buf(M)
        E = self.E
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_copy_cols_bf16(b["x"].data_ptr(), b["x"].stride(0), M, self.S, b["critic_in"][:, E:].data_ptr(),
                                                     b["critic_in"].stride(0), None, 0, self._st()), "pulse_copy_cols_bf16")
        cz = self.critic_z.forward(b["x"])
        self._reparam(cz, None, _lib.Z_MEAN, b["critic_in"], M, clamp=False)
        return self.critic.forward(b["critic_in"])

    def act(self, obs: torch.Tensor, noise: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """get_action_values in only_kin_loss mode (amp_agent.py:236-250): the env is stepped with `mus`."""
        out = self.eval_actor(obs, noise)
        if self.critic is not None:
            out["values"] = self.value_rms.unnormalize(self.eval_critic(M=obs.shape[0]))
        return out

    def act_into(self, obs: torch.Tensor, *, mus: torch.Tensor, rng_step: int = 0, noise_out: Optional[torch.Tensor] = None) -> None:
        """The student's action in the distillation rollout (get_action_values in eval mode, the env stepped with `mus`,
        amp_agent.py:359-369, amp_network_z_builder.py:82-95): normalise without a statistics update, encoder, reparameterisation
        with the noise drawn in `pulse_vae_reparam_philox` (seed, row, latent index; offset = rng_offset + rng_step), decoder writing
        `mus` (an [M, A] experience-buffer slice, any row stride).  `noise_out` fp32 [M, E] receives the draws (tests).  No critic:
        its values never reach the only_kin_loss update."""
        M = obs.shape[0]
        b = self._buf(M)
        self._normalize_obs(obs, b)
        head = self.enc.forward(b["x"])
        if noise_out is not None and (noise_out.dtype != torch.float32 or noise_out.shape != (M, self.E) or noise_out.stride(1) != 1):
            raise _lib.PulseError(f"act_into: noise_out must be float32 [{M}, {self.E}] with contiguous rows")
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_vae_reparam_philox(head.data_ptr(), head.stride(0), M, self.E, int(self.clamp), self.clamp_lo, self.clamp_hi,
                                                         self.rng_seed, self.rng_offset.data_ptr(), int(rng_step), b["dec_in"].data_ptr(),
                                                         b["dec_in"].stride(0), _lib.ptr(noise_out),
                                                         noise_out.stride(0) if noise_out is not None else 0, self._st()),
                       "pulse_vae_reparam_philox")
        self.dec.forward(b["dec_in"], out=mus)

    def advance_rng(self, steps: int) -> None:
        """Moves the device-side Philox offset past the `steps` draws of a rollout (CUDA-graph replays draw fresh noise)."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_bump_counter(self.rng_offset.data_ptr(), int(steps), self._st()), "pulse_bump_counter")

    # ------------------------------------------------------------------ update
    def anneal(self, epoch_num: int) -> float:
        """KLD annealing (amp_agent.py:827-833); call once per _optimize_kin like the reference does (after the loss)."""
        if self.kld_anneal and epoch_num > 2500:
            self.kld_coefficient = (0.01 - self.kld_coefficient_min) * max((5000 - epoch_num) / (5000 - 2500), 0) + self.kld_coefficient_min
        return self.kld_coefficient

    def optimize_kin(self, obs: torch.Tensor, gt_action: torch.Tensor, progress: torch.Tensor, noise: Optional[torch.Tensor] = None,
                     update_obs_rms: bool = False, world_size: int = 1, step: bool = True) -> torch.Tensor:
        """One AMPAgent._optimize_kin minibatch: forward, losses, explicit backward, grad-norm clip + Adam(kin_lr).
        obs fp32 [M, obs] raw (normalised here as `_preproc_obs` does), rows env-major [M/horizon, horizon]; gt_action fp32
        [M, A]; progress int64 [M].  Returns the fp64 stats tensor: [0] sum ||pred-gt||, [1] sum KL rows, [2] sum AR1 pair
        norms, [3..6] regulariser sums (losses = sums / M resp. / pairs, see `losses()`).  step=False leaves the gradients in
        `flat.grads` without the optimizer step (tests)."""
        M = obs.shape[0]
        b = self._buf(M)
        E = self.E
        main = torch.cuda.current_stream(self.device)
        if self._side is None:
            self._side = torch.cuda.Stream(self.device)
        side = self._side
        self.flat.begin_backward()
        self.stats.zero_()
        out = self.eval_actor(obs, noise, train=True, update_obs_rms=update_obs_rms)        # encoder -> z -> decoder
        side.wait_stream(main)
        with torch.cuda.stream(side):                                                        # the prior chain is independent
            prior_head = self.compute_prior(train=True, M=M)
        pred, noise = out["mus"], out["noise"]
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_vae_action_loss(pred.data_ptr(), pred.stride(0), gt_action.data_ptr(), gt_action.stride(0), M, self.A,
                                                      b["dpred"].data_ptr(), b["dpred"].stride(0), b["dpred"].shape[1], self.stats.data_ptr(),
                                                      self._st()), "pulse_vae_action_loss")
        self.dec.backward(b["dpred"], M)                                                     # also dz = dLoss/dz [M, E] fp32
        dz = self.dec._ws[(M, True)]["dx"]
        main.wait_stream(side)
        a = _lib.VaeLatentArgs(
            enc_head=out["enc_head"].data_ptr(), ld_enc=out["enc_head"].stride(0), prior_head=prior_head.data_ptr(), ld_prior=prior_head.stride(0),
            noise=noise.data_ptr(), ld_noise=noise.stride(0), dz=dz.data_ptr(), ld_dz=dz.stride(0),
            progress=progress.data_ptr() if (self.use_ar1_prior and progress is not None) else None, latent=E, horizon=self.horizon,
            clamp=int(self.clamp), clamp_lo=self.clamp_lo, clamp_hi=self.clamp_hi, kld_coef=self.kld_coefficient,
            ar1_coef=self.ar1_coefficient if self.use_ar1_prior else 0.0, regu_coef=0.005 if self.use_vae_prior_regu else 0.0, phi=0.99,
            d_enc_head=b["d_enc"].data_ptr(), ld_de=b["d_enc"].stride(0), d_prior_head=b["d_prior"].data_ptr(), ld_dp=b["d_prior"].stride(0),
            stats=self.stats[1:].data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_vae_latent_loss(C.byref(a), M, self._st()), "pulse_vae_latent_loss")
        side.wait_stream(main)
        with torch.cuda.stream(side):
            self.prior.backward(b["d_prior"], M)
        self.enc.backward(b["d_enc"], M)
        main.wait_stream(side)
        # the reference's kin_optimizer is not Horovod-wrapped (amp_agent.py:67); multi-GPU needs the average
        if world_size > 1 and step and self.flat.peer is not None:
            self.flat.peer_adam_step(self.kin_lr, max_norm=self.grad_norm)     # averaging + clip + Adam as one peer-memory kernel
        else:
            if world_size > 1:
                from .dist_utils import average_gradients
                average_gradients(self.flat.grads, world_size)
            if step:
                self.flat.adam_step(self.kin_lr, max_norm=self.grad_norm)
        return self.stats

    def losses(self, M: int) -> Dict[str, float]:
        """Host-side read-out of the last optimize_kin statistics (synchronises)."""
        s = self.stats.tolist()
        pairs = (M // self.horizon) * (self.horizon - 1)
        n = M * self.E
        out = {"kin_action_loss": s[0] / M, "kin_KLD": s[1] / M, "kin_ar1": s[2] / pairs if self.use_ar1_prior and pairs > 0 else 0.0}
        out["kin_prior_regu"] = 0.001 * (s[3] + s[4] + s[5] + s[6]) / n if self.use_vae_prior_regu else 0.0
        out["kin_loss"] = (out["kin_action_loss"] + out["kin_KLD"] * self.kld_coefficient + out["kin_ar1"] * self.ar1_coefficient
                           + out["kin_prior_regu"] * 0.005)
        return out

    # ------------------------------------------------------------------ Z-task decode (K20)
    def compute_z_actions(self, obs_buf: torch.Tensor, action_z: torch.Tensor) -> torch.Tensor:
        """HumanoidZ.compute_z_actions, z_type 'vae' + use_vae_prior: z = prior_mu(self_obs) + action_z;
        actions = decoder([clamp(self_obs, +-5), z]).  The prior sees the UNCLAMPED normalised self observation (:87 vs :147).
        obs_buf fp32 [M, >= S] raw; frozen `obs_rms` = the checkpoint's running_mean_std."""
        prior_head, dec_in = self.z_prior(obs_buf)
        self._reparam(prior_head, action_z, _lib.Z_RESIDUAL, dec_in, obs_buf.shape[0])
        return self.dec.forward(dec_in)

    def z_prior(self, obs_buf: torch.Tensor):
        """The part of compute_z_actions that does not depend on the action: the unclamped normalised self observation into the prior
        operand, the clamped one into the decoder operand's self-observation columns, the prior MLP.  Returns (prior head fp32 [M, 2E],
        decoder operand bf16 [M, Kp] whose columns [0, E) await z); `self.dec.forward(operand)` decodes."""
        M = obs_buf.shape[0]
        b = self._buf(M)
        E, S = self.E, self.S
        rms = self.obs_rms
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_normalize_cols(obs_buf.data_ptr(), obs_buf.stride(0), M, S, rms.mean_f32.data_ptr(), rms.rstd_f32.data_ptr(),
                                                     0.0, b["prior_in"].data_ptr(), b["prior_in"].stride(0), b["prior_in"].shape[1], self._st()),
                       "pulse_normalize_cols")
            _lib.check(self.lib.pulse_normalize_cols(obs_buf.data_ptr(), obs_buf.stride(0), M, S, rms.mean_f32.data_ptr(), rms.rstd_f32.data_ptr(),
                                                     5.0, b["dec_in"][:, E:].data_ptr(), b["dec_in"].stride(0), S, self._st()),
                       "pulse_normalize_cols")
        return self.prior.forward(b["prior_in"]), b["dec_in"]

    # ------------------------------------------------------------------ checkpoint keys (rl_games layout)
    def state_dict(self) -> Dict[str, torch.Tensor]:
        E = self.E
        sd = {}
        sd.update(self.enc.state_dict("z_mlp", "_zhead"))
        sd.update(self.prior.state_dict("z_prior", "_phead"))
        sd.update(self.dec.state_dict("actor_mlp", "mu"))
        for fused, mu_name, lv_name in (("_zhead", "z_mu", "z_logvar"), ("_phead", "z_prior_mu", "z_prior_logvar")):
            w, bvec = sd.pop(f"{fused}.weight"), sd.pop(f"{fused}.bias")
            sd[f"{mu_name}.weight"], sd[f"{lv_name}.weight"] = w[:E].clone(), w[E:].clone()
            sd[f"{mu_name}.bias"], sd[f"{lv_name}.bias"] = bvec[:E].clone(), bvec[E:].clone()
        if self.critic is not None:
            sd.update(self.critic_z.state_dict("critic_z_mlp", "_czhead"))
            n = 2 * (len(self.critic_z.layers) - 1)
            sd[f"critic_z_mlp.{n}.weight"], sd[f"critic_z_mlp.{n}.bias"] = sd.pop("_czhead.weight"), sd.pop("_czhead.bias")
            sd.update(self.critic.state_dict("critic_mlp", "value"))
        sd = {f"a2c_network.{k}": v for k, v in sd.items()}
        sd["a2c_network.sigma"] = self.logstd.clone()
        sd["running_mean_std.running_mean"] = self.obs_rms.running_mean.clone()
        sd["running_mean_std.running_var"] = self.obs_rms.running_var.clone()
        sd["running_mean_std.count"] = self.obs_rms.count.clone()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        s = {k[len("a2c_network."):]: v for k, v in sd.items() if k.startswith("a2c_network.")}
        s["_zhead.weight"], s["_zhead.bias"] = _split_heads(s, "z_mu", "z_logvar")
        s["_phead.weight"], s["_phead.bias"] = _split_heads(s, "z_prior_mu", "z_prior_logvar")
        self.enc.load_state_dict(s, "z_mlp", "_zhead")
        self.prior.load_state_dict(s, "z_prior", "_phead")
        self.dec.load_state_dict(s, "actor_mlp", "mu")
        if self.critic is not None and "critic_z_mlp.0.weight" in s:
            n = 2 * (len(self.critic_z.layers) - 1)
            s["_czhead.weight"], s["_czhead.bias"] = s[f"critic_z_mlp.{n}.weight"], s[f"critic_z_mlp.{n}.bias"]
            self.critic_z.load_state_dict(s, "critic_z_mlp", "_czhead")
            self.critic.load_state_dict(s, "critic_mlp", "value")
        if "sigma" in s:
            self.logstd.copy_(s["sigma"].to(self.device))
        if "running_mean_std.running_mean" in sd:
            self.obs_rms.running_mean.copy_(sd["running_mean_std.running_mean"].to(self.device).double())
            self.obs_rms.running_var.copy_(sd["running_mean_std.running_var"].to(self.device).double())
            if "running_mean_std.count" in sd:
                self.obs_rms.count.copy_(torch.as_tensor(sd["running_mean_std.count"]).to(self.device).double())
            self.obs_rms._refresh()


class TeacherPNN:
    """Frozen distillation teacher (K19): `num_prim` ReLU primitive columns (PNN without lateral links, pnn.py:127-131) and
    the composer MLP as rebuilt by `load_mcp_mlp` -- an activation after EVERY Linear including the last
    (network_loader.py:37-39) -- combined as gt_action = sum_k w_k a_k (humanoid_im_distill.py:193-198).  The input is
    normalised with the TEACHER checkpoint's running statistics and clamped to +-5 (:167-184)."""

    def __init__(self, obs_size: int = 934, num_actions: int = 69, prim_units: Sequence[int] = (1024, 512), composer_units: Sequence[int] = (1024, 512),
                 num_prim: int = 3, composer_act: str = "silu", device="cuda:0", seed: int = 0):
        self.device = torch.device(device)
        self.obs_size, self.A, self.num_prim, self.composer_act = obs_size, num_actions, num_prim, composer_act
        self.flat = FlatParams(self.device)
        self.cols = [MLP(self.flat, obs_size, list(prim_units), num_actions, "relu") for _ in range(num_prim)]
        self.composer = MLP(self.flat, obs_size, list(composer_units), num_prim, composer_act)
        self.flat.finalize(peer=False)      # frozen teacher: plain device memory
        gen = torch.Generator(device=self.device).manual_seed(seed)
        for m in self.cols + [self.composer]:
            m.init_default(gen)
        self.rms = RunningMeanStdB200(obs_size, self.device)
        self.rms.frozen = True
        self.Kp = pad_k(obs_size)
        self.lib = _lib.load()
        self._bufs: Dict[int, dict] = {}

    def load_weights(self, pnn_sd: Dict[str, torch.Tensor], composer_sd: Dict[str, torch.Tensor], running_mean: torch.Tensor,
                     running_var: torch.Tensor) -> None:
        """pnn_sd: keys `actors.<k>.<2i>.weight|bias` (PNN.state_dict()); composer_sd: `<2i>.weight|bias`."""
        def seq_keys(sd, num_layers):
            """nn.Sequential numbering (Linear at 0, 2, 4, ...) -> the prefix / head naming MLP.load_state_dict takes"""
            last = 2 * (num_layers - 1)
            out = {f"m.{k}": v for k, v in sd.items() if not k.startswith(f"{last}.")}
            out["h.weight"], out["h.bias"] = sd[f"{last}.weight"], sd[f"{last}.bias"]
            return out

        for k, col in enumerate(self.cols):
            sub = {kk[len(f"actors.{k}."):]: v for kk, v in pnn_sd.items() if kk.startswith(f"actors.{k}.")}
            col.load_state_dict(seq_keys(sub, len(col.layers)), "m", "h")
        self.composer.load_state_dict(seq_keys(composer_sd, len(self.composer.layers)), "m", "h")
        self.rms.running_mean.copy_(running_mean.to(self.device).double())
        self.rms.running_var.copy_(running_var.to(self.device).double())
        self.rms._refresh()

    def gt_action(self, obs_buf: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """obs_buf fp32 [M, obs] raw -> fp32 [M, A]: a reused buffer, or `out` (any row stride, e.g. an experience-buffer slice)."""
        M = obs_buf.shape[0]
        if M not in self._bufs:
            self._bufs[M] = {"x": torch.zeros(M, self.Kp, device=self.device, dtype=torch.bfloat16),
                             "acts": torch.zeros(self.num_prim, M, self.A, device=self.device), "out": torch.zeros(M, self.A, device=self.device)}
        b = self._bufs[M]
        self.rms.normalize_into(obs_buf, b["x"])
        for k, col in enumerate(self.cols):
            col.forward(b["x"], out=b["acts"][k])
        w = self.composer.forward(b["x"])
        if out is None:
            out = b["out"]
        elif out.dtype != torch.float32 or out.shape != (M, self.A) or out.stride(1) != 1:
            raise _lib.PulseError(f"gt_action: out must be float32 [{M}, {self.A}] with contiguous rows")
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_pnn_compose(b["acts"].data_ptr(), b["acts"].stride(0), b["acts"].stride(1), w.data_ptr(), w.stride(0),
                                                  {"silu": _lib.ACT_SILU, "relu": _lib.ACT_RELU, None: _lib.ACT_NONE}[self.composer_act], M, self.A,
                                                  self.num_prim, out.data_ptr(), out.stride(0), _lib.current_stream(self.device)),
                       "pulse_pnn_compose")
        return out


def pd_targets(actions: torch.Tensor, offset: torch.Tensor, scale: torch.Tensor, out: Optional[torch.Tensor] = None,
               freeze: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Humanoid._action_to_pd_targets (+ freeze_hand / freeze_toe zeroing), humanoid.py:1222-1247, :1392-1394 (K22).
    freeze: uint8 [dofs] mask of dofs whose target is forced to 0."""
    lib = _lib.load()
    M, D = actions.shape
    if out is None:
        out = torch.empty(M, D, device=actions.device)
    with torch.cuda.device(actions.device):
        _lib.check(lib.pulse_pd_targets(actions.data_ptr(), actions.stride(0), offset.data_ptr(), scale.data_ptr(), _lib.ptr(freeze), M, D,
                                        out.data_ptr(), out.stride(0), _lib.current_stream(actions.device)), "pulse_pd_targets")
    return out
