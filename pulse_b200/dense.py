"""Dense layers on the H100 tensor cores: thin host wrapper over `pulse_gemm_bf16` (wgmma / TMA).

`gemm_nt(a, b)` computes a @ b.T for bf16 row-major a [M,K], b [N,K] with fp32 accumulation and a fused
epilogue (bias, ReLU / SiLU, activation-derivative gating, transposed copy, fp32 output, split-K slabs).
"""
import ctypes as C
from typing import Optional

import torch

from . import _lib

ACT = {"none": _lib.ACT_NONE, None: _lib.ACT_NONE, "relu": _lib.ACT_RELU, "silu": _lib.ACT_SILU}


def _check_bf16(t, name):
    if t.dtype != torch.bfloat16 or t.dim() != 2 or t.stride(1) != 1:
        raise _lib.PulseError(f"{name} must be a 2-D bf16 tensor with contiguous rows, got {t.dtype} {tuple(t.shape)} {t.stride()}")


def num_splits(k: int, split_k: int) -> int:
    return int(_lib.load().pulse_gemm_num_splits(k, split_k))


def ordered_sum_add(x: torch.Tensor, out: torch.Tensor) -> None:
    """out += x.sum(0) for fp32 x [n, rows, cols] (rows with contiguous columns), the n terms added in order: same bits on every run."""
    if x.dtype != torch.float32 or out.dtype != torch.float32 or x.stride(-1) != 1 or out.stride(-1) != 1 or x.shape[1:] != out.shape:
        raise _lib.PulseError("ordered_sum_add: fp32 x [n, rows, cols] and out [rows, cols] with contiguous columns")
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().pulse_ordered_sum_add(x.data_ptr(), x.shape[0], x.stride(0), x.shape[1], x.shape[2], x.stride(1), out.data_ptr(),
                                                     out.stride(0), _lib.current_stream(x.device)), "pulse_ordered_sum_add")


def column_sum_add(y: torch.Tensor, out: torch.Tensor, chunk: int = 64) -> None:
    """out[c] += sum_r y[r, c] for fp32 y [rows, cols], in a fixed order (rows in chunks of `chunk`, then the chunk sums in order)."""
    rows, cols = y.shape
    n = -(-rows // chunk)
    part = torch.zeros(n, cols, device=y.device)
    full = rows // chunk
    if full:
        ordered_sum_add(y[:full * chunk].as_strided((chunk, full, cols), (y.stride(0), chunk * y.stride(0), 1)), part[:full])
    if rows > full * chunk:
        ordered_sum_add(y[full * chunk:].unsqueeze(1), part[full:])
    ordered_sum_add(part.unsqueeze(1), out.view(1, -1)[:, :cols])


def gemm_nt(a, b, **kw) -> None:
    """a [M,K] . b [N,K]^T (both K-major)."""
    gemm(a, b, **kw)


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False, bias: Optional[torch.Tensor] = None, act=None,
         gate: Optional[torch.Tensor] = None, gate_mode=None, alpha: float = 1.0, out: Optional[torch.Tensor] = None,
         out_t: Optional[torch.Tensor] = None, out_f32: Optional[torch.Tensor] = None, preact: Optional[torch.Tensor] = None,
         colsum: Optional[torch.Tensor] = None, accumulate: bool = False, split_k: int = 1, sumsq: Optional[torch.Tensor] = None,
         relu_mask: Optional[torch.Tensor] = None, gate_mask: Optional[torch.Tensor] = None) -> None:
    """D[M,N] = epilogue(sum_k A(m,k) B(n,k)).  a is [M,K] (K-major) or, with a_mn, [K,M] (MN-major: the reduction index
    is the row); likewise b is [N,K] or, with b_mn, [K,N].  No operand is ever transposed in memory.
    accumulate=True with several split-K slices: every slice writes its own fp32 slab and the slabs are added to out_f32 in slice
    order, so repeated runs give identical bits (atomic adds from concurrently running slices would not)."""
    lib = _lib.load()
    _check_bf16(a, "a")
    _check_bf16(b, "b")
    (K, M) = a.shape if a_mn else (a.shape[1], a.shape[0])
    if accumulate and out_f32 is not None and out_f32.dim() == 2 and split_k > 1 and num_splits(K, split_k) > 1:
        if (bias, gate, gate_mode, out, out_t, preact, colsum, sumsq, relu_mask, gate_mask) != (None,) * 10 or act not in (None, "none") \
                or alpha != 1.0:
            raise _lib.PulseError("split-K accumulation takes a plain fp32 output only (no alpha, activation, gate or extra outputs)")
        N = b.shape[1] if b_mn else b.shape[0]
        slabs = torch.empty(num_splits(K, split_k), M, (N + 3) // 4 * 4, device=a.device)[:, :, :N]
        gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=slabs, split_k=split_k)
        if out_f32.stride(-1) != 1:
            raise _lib.PulseError("out_f32 must be fp32 with contiguous rows")
        ordered_sum_add(slabs, out_f32[:M, :N])
        return
    (Kb, N) = b.shape if b_mn else (b.shape[1], b.shape[0])
    if K != Kb:
        raise _lib.PulseError(f"K mismatch: a {tuple(a.shape)} (mn={a_mn}) vs b {tuple(b.shape)} (mn={b_mn})")
    ep = _lib.GemmEpilogue()
    ep.alpha = alpha
    ep.act = ACT[act] if not isinstance(act, int) else act
    if bias is not None:
        if bias.dtype != torch.float32 or bias.numel() != N or not bias.is_contiguous():
            raise _lib.PulseError("bias must be contiguous fp32 [N]")
        ep.bias = bias.data_ptr()
    if gate is not None:
        _check_bf16(gate, "gate")
        ep.gate, ep.ldg = gate.data_ptr(), gate.stride(0)
        ep.gate_mode = ACT[gate_mode] if not isinstance(gate_mode, int) else gate_mode
    if out is not None:
        _check_bf16(out, "out")
        if out.shape[0] < M or out.shape[1] < N:
            raise _lib.PulseError("out too small")
        ep.out, ep.ldo = out.data_ptr(), out.stride(0)
    if out_t is not None:
        _check_bf16(out_t, "out_t")
        if out_t.shape[0] < N or out_t.shape[1] < M:
            raise _lib.PulseError("out_t too small")
        ep.out_t, ep.ldot = out_t.data_ptr(), out_t.stride(0)
    if preact is not None:
        _check_bf16(preact, "preact")
        ep.preact, ep.ldp = preact.data_ptr(), preact.stride(0)
    if out_f32 is not None:
        if out_f32.dtype != torch.float32 or out_f32.stride(-1) != 1:
            raise _lib.PulseError("out_f32 must be fp32 with contiguous rows")
        if out_f32.dim() == 3:  # [splits, M, N] slabs
            if out_f32.shape[0] < num_splits(K, split_k):
                raise _lib.PulseError("out_f32 has fewer slabs than split-K needs")
            ep.split_stride, ep.ldf = out_f32.stride(0), out_f32.stride(1)
        else:
            if split_k != 1 and not accumulate:
                raise _lib.PulseError("split_k > 1 needs a [splits, M, N] out_f32 or accumulate=True")
            ep.ldf = out_f32.stride(0)
        ep.out_f32 = out_f32.data_ptr()
        ep.accumulate = int(accumulate)
    if colsum is not None:
        if colsum.dtype != torch.float32 or colsum.numel() < N:
            raise _lib.PulseError("colsum must be fp32 [N]")
        ep.colsum = colsum.data_ptr()
    if sumsq is not None:
        if sumsq.dtype != torch.float64 or sumsq.numel() < 1:
            raise _lib.PulseError("sumsq must be an fp64 accumulator")
        ep.sumsq = sumsq.data_ptr()
    for name, t in (("relu_mask", relu_mask), ("gate_mask", gate_mask)):      # ReLU masks as bit words, [ceil(N/32), >= M] int32, chunk-major
        if t is not None:
            if t.dtype != torch.int32 or t.dim() != 2 or t.stride(1) != 1 or t.shape[0] * 32 < N or t.shape[1] < M:
                raise _lib.PulseError(f"{name} must be int32 [ceil(N/32), >= M] with contiguous rows, got {t.dtype} {tuple(t.shape)}")
            if name == "relu_mask":
                ep.relu_mask, ep.ld_rmask = t.data_ptr(), t.stride(0)
            else:
                ep.gate_mask, ep.ld_gmask = t.data_ptr(), t.stride(0)
    flags = (_lib.GEMM_A_MN if a_mn else 0) | (_lib.GEMM_B_MN if b_mn else 0)
    with torch.cuda.device(a.device):
        _lib.check(lib.pulse_gemm_bf16(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), M, N, K, C.byref(ep), split_k, flags,
                                       _lib.current_stream(a.device)), "pulse_gemm_bf16")

