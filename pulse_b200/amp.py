"""AMP discriminator on the GPU: rewards and the training loss with an ANALYTIC gradient penalty.

Host-side mirror of `AMPAgent._calc_disc_rewards` (phc/learning/amp_agent.py:1027-1041), `_disc_loss`
(:895-952) and the `eval_disc` calls of `ModelAMPContinuous.forward` (amp_models.py:33-41) for the ReLU
discriminator `AMPBuilder._build_disc` builds (amp_network_builder.py:230-249).

The reference obtains the gradient penalty's parameter gradients by double backward through
`torch.autograd.grad(..., create_graph=True)`.  For a ReLU MLP D(x) = w3 . relu(W2 relu(W1 x + b1) + b2) + b3 the
input gradient is  gx = ((m2 * w3) W2 * m1) W1  with the activation masks m1, m2 piecewise constant, so both gx
and d(mean|gx|^2)/d(W1, W2, w3) are plain GEMM chains -- the same wgmma kernel in its dgrad / wgrad / NT forms:
    g2 = m2 * w3            u = g2 W2        g1 = m1 * u        gx = g1 W1
    G  = c * gx  (c = 2 * disc_coef * grad_penalty / B)
    dW1 += g1^T G      du = m1 * (G W1^T)      dW2 += g2^T du      dw3 += colsum(m2 * (du W2^T))
"""
import ctypes as C
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .dense import column_sum_add, gemm
from .nets import MLP, FlatParams, pad_k, pick_split
from .ppo import RunningMeanStdB200


class AmpDiscriminator:
    def __init__(self, flat: FlatParams, amp_obs_size: int = 1960, units: Sequence[int] = (1024, 512), disc_coef: float = 5.0,
                 logit_reg: float = 0.01, grad_penalty: float = 5.0, weight_decay: float = 0.0001, reward_scale: float = 2.0):
        self.flat, self.device = flat, flat.device
        self.size = amp_obs_size
        self.mlp = MLP(flat, amp_obs_size, units, 1, "relu", aug=True)     # biases ride in the weights' extra column (nets.Dense)
        self.Kp = self.mlp.Kp0
        if len(units) != 2:
            raise _lib.PulseError("the analytic gradient penalty is written for the 2-hidden-layer discriminator of im.yaml")
        self.disc_coef, self.logit_reg, self.grad_penalty, self.weight_decay = disc_coef, logit_reg, grad_penalty, weight_decay
        self.reward_scale = reward_scale
        self.rms = RunningMeanStdB200(amp_obs_size, self.device)       # _amp_input_mean_std
        self.rms.pad_one = 1.0                                          # the normalised operand carries the ones column of the first layer
        self.stats = torch.zeros(8, dtype=torch.float64, device=self.device)
        self._bufs: Dict[int, dict] = {}
        self.lib = _lib.load()

    # ------------------------------------------------------------------ rewards (rollout side)
    def rewards(self, amp_obs: torch.Tensor, x_buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        """disc_r = -log(max(1 - sigmoid(D(norm(x))), 1e-4)) * disc_reward_scale   (amp_agent.py:1027-1041)."""
        R = amp_obs.shape[0]
        x = x_buf if x_buf is not None else torch.empty(R, self.Kp, device=self.device, dtype=torch.bfloat16)
        self.rms.normalize_into(amp_obs, x)
        logits = self.mlp.forward(x)
        prob = 1.0 / (1.0 + torch.exp(-logits))
        return -torch.log(torch.clamp(1.0 - prob, min=1e-4)) * self.reward_scale

    # ------------------------------------------------------------------ loss + gradients (update side)
    def _buf(self, B: int):
        if B not in self._bufs:
            dev, bf = self.device, torch.bfloat16
            L1, L2, _ = self.mlp.layers
            self._bufs[B] = {
                "x": torch.zeros(2, 3 * B, self.Kp, device=dev, dtype=bf),       # two slots: the next minibatch's operand can be prepared early
                "dlogit": torch.zeros(3 * B, 8, device=dev, dtype=bf),
                "g2": torch.zeros(B, L2.Np, device=dev, dtype=bf), "g1": torch.zeros(B, L1.Np, device=dev, dtype=bf),
                "Gb": torch.zeros(B, self.Kp, device=dev, dtype=bf),
                "du": torch.zeros(B, L1.Np, device=dev, dtype=bf), "scratch": torch.zeros(B, L2.Np, device=dev),
                "split1": pick_split(((L1.N + 127) // 128) * ((L1.Kp + 127) // 128), (B + 63) // 64),
                "split2": pick_split(((L2.N + 127) // 128) * ((L2.Kp + 127) // 128), (B + 63) // 64),
            }
        return self._bufs[B]

    def prepare_inputs(self, amp_agent: torch.Tensor, amp_replay: torch.Tensor, amp_demo: torch.Tensor, update_rms: bool = True, slot: int = 0) -> None:
        """_preproc_amp_obs in train mode for the three batches of one minibatch, in the reference's order: normalise with the current
        statistics, then merge the batch (amp_agent.py:1004-1007).  Depends on no weight, so a caller may run it for minibatch i+1
        while minibatch i is still in its backward pass / gradient all-reduce (operand `slot` = the other one)."""
        B = amp_agent.shape[0]
        if amp_replay.shape[0] != B or amp_demo.shape[0] != B:
            raise _lib.PulseError("agent / replay / demo AMP batches must have the same number of rows")
        x = self._buf(B)["x"][slot]
        for k, src in enumerate((amp_agent, amp_replay, amp_demo)):
            if update_rms:
                self.rms.normalize_update(src, x[k * B:(k + 1) * B])
            else:
                self.rms.normalize_into(src, x[k * B:(k + 1) * B])

    def loss_backward(self, amp_agent: torch.Tensor, amp_replay: torch.Tensor, amp_demo: torch.Tensor, update_rms: bool = True,
                      slot: int = 0, prepared: bool = False) -> torch.Tensor:
        """ADDS disc_coef * d(disc_loss)/d(params) into the flat gradient buffer.  Returns the fp64 stats tensor
        [sum softplus(l) agent, sum softplus(-l) demo, #agent l<0, #demo l>0, sum G^2 (G = c*gx), sum w_logit^2, sum all w^2, 0].
        `prepared`: prepare_inputs(..., slot=slot) already ran for these batches."""
        B = amp_agent.shape[0]
        if not prepared:
            self.prepare_inputs(amp_agent, amp_replay, amp_demo, update_rms, slot)
        b = self._buf(B)
        lib, dev = self.lib, self.device
        L1, L2, L3 = self.mlp.layers
        x = b["x"][slot]
        logits = self.mlp.forward(x, train=True)                      # [3B, 1]: agent, replay, demo
        self.stats.zero_()
        with torch.cuda.device(dev):
            st = _lib.current_stream(dev)
            _lib.check(lib.pulse_disc_loss(logits.data_ptr(), logits.stride(0), 2 * B, B, self.disc_coef, b["dlogit"].data_ptr(),
                                           b["dlogit"].stride(0), self.stats.data_ptr(), st), "pulse_disc_loss")
        self.mlp.backward(b["dlogit"], 3 * B)                          # prediction-loss gradients
        # ---- gradient penalty on the demo rows, analytic (see module docstring); ReLU masks = the bit words of the forward epilogue ----
        ws = self.mlp._ws[(3 * B, True)]
        h2 = ws["act"][1][2 * B:]
        m1, m2 = ws["mask"][0][:, 2 * B:], ws["mask"][1][:, 2 * B:]      # [N/32, B] views (row stride 3B) of the demo rows' masks
        w3 = L3.weight.view(-1)                                         # fp32 [Kp3]; only the first 512 are read
        with torch.cuda.device(dev):
            _lib.check(lib.pulse_relu_mask_scale(h2.data_ptr(), h2.stride(0), B, L2.N, w3.data_ptr(), b["g2"].data_ptr(), b["g2"].stride(0),
                                                 _lib.current_stream(dev)), "pulse_relu_mask_scale")
        W1, W2 = L1.w_bf16[:, :L1.K], L2.w_bf16[:, :L1.N]               # weight blocks WITHOUT the bias column
        gemm(b["g2"][:, :L2.N], W2, b_mn=True, gate_mask=m1, out=b["g1"])                                  # g1 = m1 * (g2 W2)
        c = 2.0 * self.disc_coef * self.grad_penalty / B
        gemm(b["g1"][:, :L1.N], W1, b_mn=True, alpha=c, out=b["Gb"], sumsq=self.stats[4:])                  # G = c * g1 W1, stats[4] += sum G^2
        gemm(b["g1"][:, :L1.N], b["Gb"], a_mn=True, b_mn=True, out_f32=L1.weight_grad, accumulate=True, split_k=b["split1"])  # dW1 += g1^T G (G's bias column is 0)
        gemm(b["Gb"], L1.w_bf16, gate_mask=m1, out=b["du"])                                                # du = m1 * (G W1^T); G's bias / pad columns are 0
        gemm(b["g2"][:, :L2.N], b["du"][:, :L1.N], a_mn=True, b_mn=True, out_f32=L2.weight_grad, accumulate=True, split_k=b["split2"])  # dW2 += g2^T du
        gemm(b["du"][:, :L1.N], W2, gate_mask=m2, out_f32=b["scratch"])                                    # m2 * (du W2^T), fp32
        column_sum_add(b["scratch"][:, :L2.N], L3.weight_grad.view(-1))                                    # dw3 += its column sums, fixed order
        # ---- logit regulariser and weight decay (amp_agent.py:905-908, :932-937): d/dw coef*sum(w^2) = 2*coef*w, weights only ------
        reg = _lib.WeightReg()
        reg.count = 3
        for k, l in enumerate((L1, L2, L3)):
            coef = 2.0 * self.disc_coef * (self.weight_decay + (self.logit_reg if l is L3 else 0.0))
            blk = reg.block[k]
            blk.w, blk.g, blk.rows, blk.cols, blk.ld, blk.coef = l.weight.data_ptr(), l.weight_grad.data_ptr(), l.N, l.K, l.Kp, coef
            blk.sumsq = self.stats[6:].data_ptr()
            if l is L3:
                blk.sumsq2 = self.stats[5:].data_ptr()
        with torch.cuda.device(dev):
            _lib.check(lib.pulse_weight_reg(C.byref(reg), _lib.current_stream(dev)), "pulse_weight_reg")
        return self.stats

    def loss_from_stats(self, stats: torch.Tensor, B: int) -> Dict[str, float]:
        """Assemble the reference's scalar outputs from the device statistics (one D2H copy, logging only)."""
        s = stats.cpu()
        c = 2.0 * self.disc_coef * self.grad_penalty / B
        gp = float(s[4]) / (c * c) / B
        bce = 0.5 * (float(s[0]) / (2 * B) + float(s[1]) / B)
        loss = bce + self.logit_reg * float(s[5]) + self.grad_penalty * gp + self.weight_decay * float(s[6])
        return {"disc_loss": loss, "disc_grad_penalty": gp, "disc_logit_loss": float(s[5]), "disc_agent_acc": float(s[2]) / (2 * B),
                "disc_demo_acc": float(s[3]) / B}

    def loss_tensors(self, B: int) -> Dict[str, torch.Tensor]:
        """The entries `AMPAgent._disc_loss` returns (amp_agent.py:939-952) as DEVICE tensors from the statistics of the last
        loss_backward call (no host synchronisation; the mean logits are read from the logits that call left in the workspace)."""
        s = self.stats
        c = 2.0 * self.disc_coef * self.grad_penalty / B
        gp = s[4] / (c * c) / B
        bce = 0.5 * (s[0] / (2 * B) + s[1] / B)
        logits = self.mlp._ws[(3 * B, True)]["out"]
        return {"disc_loss": bce + self.logit_reg * s[5] + self.grad_penalty * gp + self.weight_decay * s[6], "disc_grad_penalty": gp,
                "disc_logit_loss": s[5].clone(), "disc_agent_acc": s[2] / (2 * B), "disc_demo_acc": s[3] / B,
                "disc_agent_logit": logits[:2 * B].mean(), "disc_demo_logit": logits[2 * B:].mean()}

    def state_dict(self) -> Dict[str, torch.Tensor]:
        sd = {f"a2c_network.{k}": v for k, v in self.mlp.state_dict("_disc_mlp", "_disc_logits").items()}
        sd["amp_input_mean_std.running_mean"] = self.rms.running_mean.clone()
        sd["amp_input_mean_std.running_var"] = self.rms.running_var.clone()
        sd["amp_input_mean_std.count"] = self.rms.count.clone()
        return sd
