"""MLP stacks of the PULSE / PHC agents on the H100 tensor cores.

Mirrors what `phc.learning.network_builder.NetworkBuilder._build_mlp` + `AMPBuilder.Network`
(network_builder.py:105-124, amp_network_builder.py:20-249) build -- Linear+activation stacks with a
linear head -- but stores them for the wgmma GEMM: fp32 master weights in ONE flat buffer (so the
gradient all-reduce, the norm clip and Adam are single launches) with a bf16 mirror in the same
layout that the Adam kernel writes -- the GEMM operands.  Nothing is ever transposed in memory: the
GEMM reads K-major or MN-major operands as they sit (forward: X, W K-major; dgrad: dY K-major, W
MN-major; wgrad: dY, X MN-major).

Forward / backward are explicit (no autograd): forward Y = act(X W^T + b); dgrad dX = (dY W) * act'(.)
with the bias gradient of the layer below (column sums of dX) fused into its epilogue; wgrad
dW = dY^T X accumulated with fp32 atomics across split-K CTAs straight into the flat gradient buffer.
"""
import ctypes as C
import math
import os
import warnings
from typing import Dict, List, Optional, Sequence

import torch

from . import _lib
from .dense import gemm, gemm_nt


def pad8(n: int) -> int:
    return (n + 7) // 8 * 8


def pad_k(n: int) -> int:
    """Leading dimension of a GEMM operand with n useful columns: a multiple of 64 bf16 (128 bytes) once n > 64, so every
    64-column TMA box row starts on a 128-byte line (a 936-wide row makes each box row straddle an extra 32-byte sector)."""
    return pad8(n) if n <= 64 else (n + 63) // 64 * 64


def pick_split(tiles: int, num_kb: int, sms: int = 132, epilogue_kb: int = 24) -> int:
    """Split-K factor for a weight-gradient GEMM on the persistent kernel: minimise rounds x (k-blocks per item +
    epilogue cost in k-block equivalents), where rounds = ceil(tiles * splits / SMs)."""
    best, best_cost = 1, None
    for s in range(1, min(64, num_kb) + 1):
        per = -(-num_kb // s)
        if -(-num_kb // per) != s:
            continue  # not every slice would get a k-block
        rounds = -(-(tiles * s) // sms)
        cost = rounds * (per + epilogue_kb)
        if best_cost is None or cost < best_cost:
            best, best_cost = s, cost
    return best


class FlatParams:
    """One flat fp32 buffer each for parameters, gradients and the two Adam moments."""

    def __init__(self, device):
        self.device = device
        self._shapes: List[tuple] = []
        self._numel = 0
        self.params = self.grads = self.exp_avg = self.exp_avg_sq = None
        self.step = None   # device-side Adam step counter (keeps the update CUDA-graph replayable)
        self.sumsq = None

    def reserve(self, *shape) -> int:
        off = self._numel
        n = 1
        for s in shape:
            n *= s
        self._numel += (n + 63) // 64 * 64  # every tensor 128-byte aligned in the bf16 operand buffer (TMA box rows on line starts)
        self._shapes.append((off, tuple(shape)))
        return len(self._shapes) - 1

    def finalize(self, peer: Optional[bool] = None):
        """Allocates the flat buffers.  `peer` (default: PULSE_PEER_ADAM != 0 and an initialised NCCL process group with more than one
        rank): gradients, fp32 masters and the bf16 operands live in symmetric memory mapped into every rank of the node, so the
        optimizer step is pulse_peer_reduce_adam (csrc/peer_adam.cu) instead of NCCL all-reduce + sum_squares + Adam; the Adam moments
        are then SHARDED (rank r keeps slice r current; gather_moments() before reading them).  COLLECTIVE when peer mode is on: every
        rank finalises its FlatParams objects in the same order."""
        z = lambda: torch.zeros(self._numel, device=self.device, dtype=torch.float32)
        self.peer = None
        if peer is None:
            peer = os.environ.get("PULSE_PEER_ADAM", "1") != "0"
        if peer and torch.device(self.device).type == "cuda":
            try:
                self._alloc_peer()
            except Exception as e:   # no symmetric memory on this box / driver: NCCL path (same results up to summation order)
                warnings.warn(f"pulse_b200: peer-memory optimizer unavailable ({type(e).__name__}: {e}); using the NCCL all-reduce path")
                self.peer = None
        if self.peer is None:
            self.params, self.grads = z(), z()
            self.params_bf16 = torch.zeros(self._numel, device=self.device, dtype=torch.bfloat16)
        self.exp_avg, self.exp_avg_sq = z(), z()
        self.sumsq = torch.zeros(1, device=self.device, dtype=torch.float64)
        self.step = torch.zeros(1, device=self.device, dtype=torch.int32)
        self._adam_sync = torch.zeros(1, device=self.device, dtype=torch.int32)   # last-block counter of the self-contained Adam launch
        self.clean = True                                                          # gradients are all zero

    # ------------------------------------------------------------------ peer-memory optimizer (multi-GPU)
    def _alloc_peer(self):
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() <= 1 or dist.get_backend() != "nccl":
            return
        world, rank = dist.get_world_size(), dist.get_rank()
        if world > _lib.PEER_MAX:
            return
        import torch.distributed._symmetric_memory as symm
        group = dist.group.WORLD
        try:
            symm.enable_symm_mem_for_group(group.group_name)
        except Exception:
            pass

        def alloc(n, dtype):
            t = symm.empty(n, dtype=dtype, device=self.device)
            t.zero_()
            return t, symm.rendezvous(t, group)

        grads, hg = alloc(self._numel, torch.float32)
        params, hp = alloc(self._numel, torch.float32)
        pbf16, hb = alloc(self._numel, torch.bfloat16)
        sig, hs = alloc(256, torch.uint8)
        torch.cuda.synchronize(self.device)
        dist.barrier()                                   # every rank's buffers are zeroed before anyone can signal into them
        a = _lib.PeerAdamArgs(rank=rank, world=world, count=self._numel)
        for p in range(world):
            a.grads[p], a.params[p], a.params_bf16[p], a.signals[p] = int(hg.buffer_ptrs[p]), int(hp.buffer_ptrs[p]), int(hb.buffer_ptrs[p]), int(hs.buffer_ptrs[p])
        if int(a.grads[rank]) != grads.data_ptr() or int(a.params[rank]) != params.data_ptr():
            raise RuntimeError("symmetric-memory handle does not describe the local tensors")
        # multimem (NVLS) variant by default at 8 ranks: the switch-side reduction pays once the peer count makes the pull / push
        # fan-out the bound
        mc_env = os.environ.get("PULSE_PEER_MC", "auto")
        use_mc = mc_env == "1" or (mc_env == "auto" and world >= 8)
        mc = [int(getattr(h, "multicast_ptr", 0) or 0) for h in (hg, hp, hb)]
        if use_mc and all(mc):
            a.mc_grads, a.mc_params, a.mc_params_bf16 = mc
        self.grads, self.params, self.params_bf16 = grads, params, pbf16
        dev = self.device
        scratch = dict(epoch=torch.zeros(1, dtype=torch.int32, device=dev), partials=torch.zeros(_lib.PEER_MAX_GRID, dtype=torch.float64, device=dev),
                       bar=torch.zeros(1, dtype=torch.int64, device=dev))
        a.epoch, a.cta_partials, a.grid_bar = scratch["epoch"].data_ptr(), scratch["partials"].data_ptr(), scratch["bar"].data_ptr()
        a.grid = int(os.environ.get("PULSE_PEER_GRID", "0"))
        a.timeout_ms = int(os.environ.get("PULSE_PEER_TIMEOUT_MS", "0"))     # 0 = the library default (30 min, see csrc/peer_adam.cu)
        self.peer = dict(args=a, handles=(hg, hp, hb, hs), signals=sig, scratch=scratch, world=world, rank=rank, multicast=bool(a.mc_grads))

    def shard_span(self):
        """[start, end) elements of the flat buffers whose Adam moments THIS rank keeps current in peer mode."""
        if self.peer is None:
            return 0, self._numel
        w, r, n4 = self.peer["world"], self.peer["rank"], self._numel // 4
        per = (n4 + w - 1) // w
        s0 = min(per * r, n4)
        return 4 * s0, 4 * min(s0 + per, n4)

    def peer_adam_step(self, lr: float, max_norm: float = 0.0, betas=(0.9, 0.999), eps: float = 1e-8):
        """Gradient averaging over the ranks + clip_grad_norm_ + Adam + operand refresh + gradient clearing as one launch per rank
        (hvd.DistributedOptimizer + amp_agent.py:725-750).  Every rank must call it (the kernel waits for its peers)."""
        a = self.peer["args"]
        a.exp_avg, a.exp_avg_sq, a.step = self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), self.step.data_ptr()
        a.max_norm, a.lr, a.beta1, a.beta2, a.eps = float(max_norm or 0.0), float(lr), float(betas[0]), float(betas[1]), float(eps)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pulse_peer_reduce_adam(C.byref(a), _lib.current_stream(self.device)), "pulse_peer_reduce_adam")
        self.clean = True

    def gather_moments(self):
        """Peer mode shards the Adam moments: bring every rank's copy up to date (checkpoints, tests).  Collective."""
        if self.peer is None:
            return
        import torch.distributed as dist
        s0, s1 = self.shard_span()
        for buf in (self.exp_avg, self.exp_avg_sq):
            tmp = torch.zeros_like(buf)
            tmp[s0:s1] = buf[s0:s1]
            dist.all_reduce(tmp)
            buf.copy_(tmp)

    def sync_bf16(self):
        """bf16 mirror <- fp32 masters (after init / checkpoint load; the Adam kernel keeps it current afterwards)."""
        self.params_bf16.copy_(self.params)

    def view(self, idx: int, what: str = "params") -> torch.Tensor:
        off, shape = self._shapes[idx]
        n = 1
        for s in shape:
            n *= s
        return getattr(self, what)[off:off + n].view(*shape)

    def view_padded(self, idx: int, what: str, n: int) -> torch.Tensor:
        """first n elements of slot idx INCLUDING its alignment padding (slots are padded to multiples of 64)."""
        off, _ = self._shapes[idx]
        return getattr(self, what)[off:off + n]

    def offset(self, idx: int) -> int:
        """first element of slot idx in the flat buffers"""
        return self._shapes[idx][0]

    @property
    def numel(self):
        return self._numel

    def slot_span(self, first_idx: int, last_idx: int):
        """[start, end) element range of the flat buffers covered by slots first_idx .. last_idx (alignment padding included)."""
        start = self._shapes[first_idx][0]
        end = self._shapes[last_idx + 1][0] if last_idx + 1 < len(self._shapes) else self._numel
        return start, end

    def zero_grad(self):
        self.grads.zero_()
        self.clean = True

    def begin_backward(self):
        """Called once per minibatch before gradients are accumulated: clears the buffer only if the last accumulation was not followed by
        an optimizer step (adam_step leaves the gradients zeroed -- the kernel clears what it consumed)."""
        if not self.clean:
            self.grads.zero_()
        self.clean = False

    def adam_step(self, lr: float, max_norm: float = 0.0, betas=(0.9, 0.999), eps: float = 1e-8, zero_grads: bool = True):
        """nn.utils.clip_grad_norm_(max_norm) + torch.optim.Adam step (amp_agent.py:725-750): the gradient-norm pass and ONE Adam launch that
        also advances the device-side step counter, re-zeroes the norm accumulator and clears the consumed gradients; no host sync."""
        lib = _lib.load()
        with torch.cuda.device(self.device):
            st = _lib.current_stream(self.device)
            sumsq_ptr = None
            if max_norm and max_norm > 0:
                _lib.check(lib.pulse_sum_squares(self.grads.data_ptr(), self._numel, self.sumsq.data_ptr(), st), "pulse_sum_squares")
                sumsq_ptr = self.sumsq.data_ptr()
            _lib.check(lib.pulse_adam_step(self.params.data_ptr(), self.grads.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
                                           self._numel, sumsq_ptr, float(max_norm or 0.0), lr, betas[0], betas[1], eps, self.step.data_ptr(),
                                           self.params_bf16.data_ptr(), 3 if zero_grads else 2, self._adam_sync.data_ptr(), st),
                       "pulse_adam_step")
        self.clean = bool(zero_grads)


class Dense:
    """One Linear layer.  Plain: W [N, Kp] (K padded with zero columns, see pad_k) and b [N] as separate slots.
    Bias-augmented (`aug`): ONE slot W [N, Kp] with Kp = pad_k(K + 1) whose column K holds the bias; the operand it multiplies carries
    1.0 in its column K (written by the normalise kernels / set once in the activation buffers), so the bias add of the forward pass
    and the bias gradient of the backward pass (column K of dW = dY^T [X | 1]) are done by the tensor cores -- no bias loads in the
    forward epilogue, no column sums in the dgrad epilogue."""

    def __init__(self, flat: FlatParams, in_features: int, out_features: int, act: Optional[str], aug: bool = False):
        self.K, self.N, self.act, self.aug = in_features, out_features, act, aug
        self.Kp = pad_k(in_features + 1) if aug else pad_k(in_features)
        self.Np = pad_k(out_features + 1) if aug else pad_k(out_features)    # width of this layer's OUTPUT buffer (= the next layer's Kp)
        self.flat = flat
        self.w_idx = flat.reserve(out_features, self.Kp)
        self.b_idx = None if aug else flat.reserve(out_features)
        self.ref_cols = None   # LongTensor [K]: reference input column j sits in internal column ref_cols[j] (None: the same order)

    # views (valid after flat.finalize())
    @property
    def weight(self):
        return self.flat.view(self.w_idx)

    @property
    def bias(self):
        return self.weight[:, self.K] if self.aug else self.flat.view(self.b_idx)

    @property
    def w_bf16(self):
        return self.flat.view(self.w_idx, "params_bf16")

    @property
    def weight_grad(self):
        return self.flat.view(self.w_idx, "grads")

    @property
    def bias_grad(self):
        return self.weight_grad[:, self.K] if self.aug else self.flat.view(self.b_idx, "grads")

    @property
    def pad_start(self):
        """first column of the weight matrix that must stay exactly zero"""
        return self.K + (1 if self.aug else 0)

    def init_default(self, gen: Optional[torch.Generator] = None):
        """torch.nn.Linear default init (kaiming_uniform(a=sqrt(5)) -> U(-1/sqrt(K), 1/sqrt(K)) for W and b)."""
        bound = 1.0 / math.sqrt(self.K)
        w = (torch.rand(self.N, self.K, device=self.flat.device, generator=gen) * 2 - 1) * bound
        b = (torch.rand(self.N, device=self.flat.device, generator=gen) * 2 - 1) * bound
        self.set_weights(w, b)

    def ref_weight(self, what: str = "params") -> torch.Tensor:
        """Copy of the weight block [N, K] of a weight-shaped slot (parameters, gradients or an Adam moment) in the reference's
        input-column order."""
        m = self.flat.view(self.w_idx, what)
        return m[:, :self.K].clone() if self.ref_cols is None else m[:, self.ref_cols.to(m.device)]

    def set_ref_weight(self, what: str, w: torch.Tensor) -> None:
        """Inverse of ref_weight: writes a reference-ordered [N, K] block into the slot."""
        m = self.flat.view(self.w_idx, what)
        if self.ref_cols is None:
            m[:, :self.K].copy_(w)
        else:
            m[:, self.ref_cols.to(m.device)] = w.to(m.device, m.dtype)

    def set_weights(self, w: torch.Tensor, b: torch.Tensor):
        self.weight.zero_()
        self.set_ref_weight("params", w)
        self.bias.copy_(b)
        self.refresh()

    def refresh(self):
        """bf16 operand copy of this layer (init / load path; Adam maintains it during training)."""
        self.w_bf16.copy_(self.weight)


class MLP:
    """units: hidden sizes; `head` linear output layer size, or None for a headless net whose last layer keeps its activation and
    writes bf16 (forward(out=) may give it a window of a caller's operand, e.g. the task encoder writing into the policy input).
    Activation 'relu' | 'silu'.
    hidden_acts: per-hidden-layer override (None = a Linear with no activation, e.g. the last Linear of `z_mlp` that feeds the
    `z_mu` / `z_logvar` heads, amp_network_z_builder.py:492-497).  input_grad_cols > 0: backward() also returns the gradient
    w.r.t. the first `input_grad_cols` input columns (the latent window of the PULSE decoder input).
    in_perm: internal input column i holds reference input column in_perm[i] (checkpoint import / export of layer 0).
    aug: bias-augmented layers (see Dense) -- the caller's input operand must carry 1.0 in column `in_features`.
    ReLU layers save their activation masks as bit words in the forward epilogue (train=True) and the backward pass gates with those.
    first: layer 0, reserved by the caller (so that two nets' first layers can sit back to back in the flat buffers)."""

    def __init__(self, flat: FlatParams, in_features: int, units: Sequence[int], head: Optional[int], act: str = "relu",
                 hidden_acts: Optional[Sequence[Optional[str]]] = None, input_grad_cols: int = 0, in_perm: Optional[torch.Tensor] = None,
                 aug: bool = False, first: Optional[Dense] = None):
        self.flat = flat
        self.act = act
        self.aug = aug
        self.headless = head is None
        sizes = [in_features] + list(units)
        acts = list(hidden_acts) if hidden_acts is not None else [act] * len(units)
        if len(acts) != len(units):
            raise _lib.PulseError("hidden_acts must have one entry per hidden layer")
        if first is not None and (first.K, first.N, first.act, first.aug) != (in_features, sizes[1], acts[0], aug):
            raise _lib.PulseError("the caller-reserved first layer does not match the net's input size, width, activation or bias layout")
        self.layers: List[Dense] = [first if (i == 0 and first is not None) else Dense(flat, sizes[i], sizes[i + 1], acts[i], aug)
                                    for i in range(len(units))]
        if head is not None:
            self.layers.append(Dense(flat, sizes[-1], head, None, aug))
        self.in_features, self.Kp0 = in_features, self.layers[0].Kp
        self.input_grad_cols = input_grad_cols
        self.in_perm = in_perm
        self._ws: Dict[int, dict] = {}
        self._dact0: Dict[int, torch.Tensor] = {}
        self._scratch = None
        self._zero = None

    def param_span(self):
        """[start, end) of this network's parameters / gradients inside the flat buffers (its layers are reserved back to back)."""
        idx = [i for l in self.layers for i in (l.w_idx, l.b_idx) if i is not None]
        return self.flat.slot_span(min(idx), max(idx))

    def _zero_bias(self) -> torch.Tensor:
        """read-only zeros: the `bias` argument of the fused single-output-head kernel when the bias lives in the weight row"""
        if self._zero is None:
            self._zero = torch.zeros(8, device=self.flat.device)
        return self._zero

    def init_default(self, gen=None):
        for l in self.layers:
            l.init_default(gen)

    def refresh(self):
        for l in self.layers:
            l.refresh()

    def _workspace(self, M: int, train: bool, slot: int = 0):
        key = (M, train) if slot == 0 else (M, train, slot)      # slot > 0: a second evaluation workspace for a concurrent forward pass
        if key not in self._ws:
            dev = self.flat.device
            bf = lambda r, c: torch.zeros(r, c, device=dev, dtype=torch.bfloat16)
            ws = {"act": [], "pre": [], "dact": [], "split": [], "mask": []}
            for i, l in enumerate(self.layers):
                last = i == len(self.layers) - 1
                fp32_head = last and not self.headless
                a = None if fp32_head else bf(M, l.Np)
                if a is not None and self.aug:
                    a[:, l.N] = 1.0                    # the ones column the next (bias-augmented) layer multiplies its bias column with
                ws["act"].append(a)
                if train:
                    ws["pre"].append(bf(M, l.Np) if (l.act == "silu") else None)
                    if i == 0 and not last and M in self._dact0:
                        ws["dact"].append(self._dact0[M])
                    else:
                        ws["dact"].append(None if last else bf(M, l.Np))      # gradient w.r.t. this layer's OUTPUT
                    ws["mask"].append(torch.zeros((l.N + 31) // 32, M, device=dev, dtype=torch.int32) if (l.act == "relu" and not fp32_head) else None)
                    tiles = ((l.N + 127) // 128) * ((l.Kp + 127) // 128)   # 128 x 128 output tiles
                    ws["split"].append(pick_split(tiles, (M + 63) // 64))
            hn = self.layers[-1].N     # fp32 head output: rows padded to a multiple of 4 floats so the epilogue's 16-byte stores apply (N = 69)
            ws["out"] = torch.zeros(M, (hn + 3) // 4 * 4, device=dev)[:, :hn]
            if train and self.input_grad_cols:
                ws["dx"] = torch.zeros(M, self.input_grad_cols, device=dev)
            self._ws[key] = ws
        return self._ws[key]

    def provide_dact0(self, M: int, buf: torch.Tensor) -> None:
        """Training at batch size M writes the gradient w.r.t. layer 0's pre-activation into `buf` (bf16 [M, >= N0], any row stride)
        instead of a buffer of its own: two nets can then fill the two column halves of ONE operand."""
        if buf.dtype != torch.bfloat16 or buf.shape[0] != M or buf.shape[1] < self.layers[0].N or buf.stride(1) != 1:
            raise _lib.PulseError("provide_dact0: bf16 [M, >= N0] with contiguous rows")
        self._dact0[M] = buf
        if (M, True) in self._ws:
            self._ws[(M, True)]["dact"][0] = buf

    def top_preact(self, M: int) -> torch.Tensor:
        """SiLU pre-activation of a headless net's last layer from the last training forward pass at batch size M (the gate of the
        gradient a caller hands to backward())."""
        return self._ws[(M, True)]["pre"][-1]

    def _dummy(self, n: int) -> torch.Tensor:
        """fp32 scratch the fused single-output-head kernels may add bias gradients into when the layers are bias-augmented (the weight
        gradients already contain them); never read."""
        if self._scratch is None or self._scratch.numel() < n:
            self._scratch = torch.zeros(max(n, 8), device=self.flat.device)
        return self._scratch

    def _head1(self, i: int) -> bool:
        """Layer i is a single-output head on top of a ReLU layer narrow enough for the fused GEMV kernels."""
        l = self.layers[i]
        return not self.headless and i == len(self.layers) - 1 and i > 0 and l.N == 1 and self.layers[i - 1].act == "relu" and l.Kp <= 2048

    # ---- per-layer GEMM arguments ------------------------------------------------------------------------------------------------
    def _fwd_problem(self, i: int, h: torch.Tensor, ws: dict, train: bool):
        l = self.layers[i]
        kw = dict(bias=None if self.aug else l.bias, act=l.act, out=ws["act"][i], preact=ws["pre"][i] if train else None)
        if train and ws["mask"][i] is not None:
            kw["relu_mask"] = ws["mask"][i]
        return h[:, :l.Kp], l.w_bf16, kw

    def _wgrad_problem(self, i: int, dy: torch.Tensor, x_in: torch.Tensor, ws: dict):
        l = self.layers[i]
        # dW [N, Kp] += dY^T . X, both operands MN-major (reduction over the batch rows), fp32 atomics across split-K; with augmented
        # layers X carries the ones column, so column K of dW IS the bias gradient
        return dy[:, :l.N], x_in[:, :l.Kp], dict(a_mn=True, b_mn=True, out_f32=l.weight_grad, accumulate=True, split_k=ws["split"][i])

    def _dgrad_problem(self, i: int, dy: torch.Tensor, ws: dict):
        """dX [M, K] = dY [M, N] . W [N, K] (W read MN-major), gated by act'(.) of the layer below."""
        l, prev = self.layers[i], self.layers[i - 1]
        kw = dict(b_mn=True, out=ws["dact"][i - 1])
        if prev.act == "relu" and ws["mask"][i - 1] is not None:
            kw["gate_mask"] = ws["mask"][i - 1]
        elif prev.act is not None:
            kw.update(gate=ws["pre"][i - 1] if prev.act == "silu" else ws["act"][i - 1], gate_mode=prev.act)
        if not self.aug:   # plain layers: the epilogue also accumulates the bias gradient of the layer below (column sums of dX)
            kw["colsum"] = self.flat.view_padded(prev.b_idx, "grads", prev.Np)
        w = l.w_bf16[:, :prev.N] if self.aug else l.w_bf16       # augmented: never differentiate through the bias column
        return dy[:, :l.N], w, kw

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor, train: bool = False, out: Optional[torch.Tensor] = None, slot: int = 0) -> torch.Tensor:
        """x: bf16 [M, Kp0] (normalised, zero padded; column `in_features` = 1.0 for augmented nets).  Returns fp32 [M, head] (view of a
        reused workspace buffer, or `out`).  With train=True the activations / ReLU masks / SiLU pre-activations backward() needs are kept.
        Headless nets return the bf16 activation of the last layer: columns [0, N) of `out` when given (any row stride), else of a
        workspace buffer."""
        M = x.shape[0]
        ws = self._workspace(M, train, slot)
        if out is not None and not self.headless:
            ws = dict(ws, out=out)
        h = x
        for i, l in enumerate(self.layers):
            last = i == len(self.layers) - 1
            if last and self.headless:
                a, b, kw = self._fwd_problem(i, h, ws, train)
                if out is not None:
                    kw["out"] = out
                gemm_nt(a, b, **kw)
                h = kw["out"]
            elif last and self._head1(i):
                # [M,K] x [K,1]: no tensor-core shape -- one HBM pass over h (pulse_head1_forward); augmented: the bias is w[K] * h[:, K]
                bias = self._zero_bias() if self.aug else l.bias
                with torch.cuda.device(self.flat.device):
                    _lib.check(_lib.load().pulse_head1_forward(h.data_ptr(), h.stride(0), M, l.Kp, l.w_bf16.data_ptr(), bias.data_ptr(),
                                                               ws["out"].data_ptr(), ws["out"].stride(0),
                                                               _lib.current_stream(self.flat.device)), "pulse_head1_forward")
            elif last:
                gemm_nt(h[:, :l.Kp], l.w_bf16, bias=None if self.aug else l.bias, act=None, out_f32=ws["out"])
            else:
                a, b, kw = self._fwd_problem(i, h, ws, train)
                gemm_nt(a, b, **kw)
                h = ws["act"][i]
        if train:
            self._ws[(M, True)]["x"] = x
        return h[:, :self.layers[-1].N] if self.headless else ws["out"]

    # ------------------------------------------------------------------ backward
    def _backward_head(self, ws: dict, dout: torch.Tensor, M: int):
        """Head layer: returns (dy, top) = gradient w.r.t. the output of layer `top` still to be propagated."""
        lib = _lib.load()
        dev = self.flat.device
        head = self.layers[-1]
        top = len(self.layers) - 1
        if self._head1(top):
            # single-output head: bias gradient, weight gradient, gated input gradient and the bias gradient of the layer
            # below in ONE pass over the last hidden activation (replaces a column sum and three degenerate GEMMs)
            prev, h, dh = self.layers[top - 1], ws["act"][top - 1], ws["dact"][top - 1]
            if self.aug:
                hb, pb = self._dummy(prev.Np + 8), self._dummy(prev.Np + 8)[8:]
            else:
                hb, pb = head.bias_grad, self.flat.view_padded(prev.b_idx, "grads", prev.Np)
            with torch.cuda.device(dev):
                if "head1_partials" not in ws:
                    ws["head1_partials"] = torch.empty(_lib.HEAD1_MAX_CTAS * (2 * head.Kp + 1), device=dev)
                _lib.check(lib.pulse_head1_backward(h.data_ptr(), h.stride(0), M, head.Kp, dout.data_ptr(), dout.stride(0), head.w_bf16.data_ptr(),
                                                    dh.data_ptr(), dh.stride(0), head.weight_grad.data_ptr(), hb.data_ptr(), pb.data_ptr(),
                                                    ws["head1_partials"].data_ptr(), _lib.current_stream(dev)), "pulse_head1_backward")
            return dh, top - 1
        if not self.aug:
            with torch.cuda.device(dev):  # bias gradient of the head: column sums of dout
                _lib.check(lib.pulse_column_sum_bf16(dout.data_ptr(), dout.stride(0), M, head.N, head.bias_grad.data_ptr(), _lib.current_stream(dev)),
                           "pulse_column_sum_bf16")
        return dout, top

    def backward(self, dout: torch.Tensor, M: int) -> None:
        """dout bf16 [M, pad8(head)]: gradient of the loss w.r.t. the head output (headless nets: w.r.t. the last layer's
        PRE-activation, i.e. already gated by its activation's derivative).  ADDS dW, db of every layer into the flat gradient buffer
        (the caller zeroes it once per minibatch with flat.zero_grad())."""
        ws = self._ws[(M, True)]
        dy, top = self._backward_head(ws, dout, M)
        for i in reversed(range(top + 1)):
            l = self.layers[i]
            x_in = ws["x"] if i == 0 else ws["act"][i - 1]
            a, b, kw = self._wgrad_problem(i, dy, x_in, ws)
            gemm(a, b, **kw)
            if i > 0:
                a, b, kw = self._dgrad_problem(i, dy, ws)
                gemm(a, b, **kw)
                dy = ws["dact"][i - 1]
            elif self.input_grad_cols:
                # gradient w.r.t. the leading input columns only: dX[:, :c] = dY . W[:, :c]
                gemm(dy[:, :l.N], l.w_bf16[:, :self.input_grad_cols], b_mn=True, out_f32=ws["dx"])

    # ------------------------------------------------------------------ checkpoint names
    def state_dict(self, prefix: str, head_name: Optional[str] = None) -> Dict[str, torch.Tensor]:
        """rl_games / nn.Sequential naming: `<prefix>.<2*i>.weight` for hidden layers, `<head_name>.weight` for the head."""
        out = {}
        hidden = self.layers[:-1] if head_name is not None else self.layers
        for i, l in enumerate(hidden):
            w = l.weight[:, :l.K].clone()
            if i == 0 and self.in_perm is not None:
                w_ref = torch.empty_like(w)
                w_ref[:, self.in_perm.to(w.device)] = w
                w = w_ref
            out[f"{prefix}.{2 * i}.weight"] = w
            out[f"{prefix}.{2 * i}.bias"] = l.bias.clone()
        if head_name is not None:
            l = self.layers[-1]
            out[f"{head_name}.weight"] = l.weight[:, :l.K].clone()
            out[f"{head_name}.bias"] = l.bias.clone()
        return out

    def load_state_dict(self, sd: Dict[str, torch.Tensor], prefix: str, head_name: Optional[str] = None):
        hidden = self.layers[:-1] if head_name is not None else self.layers
        for i, l in enumerate(hidden):
            w = sd[f"{prefix}.{2 * i}.weight"].to(self.flat.device)
            if i == 0 and self.in_perm is not None:
                w = w[:, self.in_perm.to(w.device)]
            l.set_weights(w, sd[f"{prefix}.{2 * i}.bias"].to(self.flat.device))
        if head_name is not None:
            l = self.layers[-1]
            l.set_weights(sd[f"{head_name}.weight"].to(self.flat.device), sd[f"{head_name}.bias"].to(self.flat.device))


def normalize_to_bf16(x: torch.Tensor, mean: Optional[torch.Tensor], rstd: Optional[torch.Tensor], out: torch.Tensor,
                      out_t: Optional[torch.Tensor] = None, pad_one: float = 0.0) -> None:  # out_t: optional transposed copy (not used by the MLPs any more)
    """RunningMeanStd eval path (running_mean_std.py:69-95) fused with the bf16 cast / zero pad / transpose.  pad_one = 1.0 writes the
    "ones" column of a bias-augmented operand into the first pad column."""
    lib = _lib.load()
    rows, cols = x.shape
    if x.dtype != torch.float32 or x.stride(1) != 1:
        raise _lib.PulseError("normalize_to_bf16: x must be fp32 with contiguous rows")
    with torch.cuda.device(x.device):
        _lib.check(lib.pulse_normalize_to_bf16(x.data_ptr(), x.stride(0), rows, cols, _lib.ptr(mean), _lib.ptr(rstd), out.data_ptr(), out.stride(0),
                                               _lib.ptr(out_t), out_t.stride(0) if out_t is not None else 0, float(pad_one),
                                               _lib.current_stream(x.device)),
                   "pulse_normalize_to_bf16")

