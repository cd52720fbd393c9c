"""Teacher-forced float64 references of the update's links, each with its own rounding bound.

A link is one GEMM or one element-wise kernel of the update.  Its reference is recomputed in float64 from the operands the kernels
themselves produced and stored (the bf16 activations, mask words and gradients in the workspaces, the bf16 weight mirror as it was
before the call), so an error in one link does not propagate into the next and every link can be held to a tight bound:

* GEMM, fp32 output:  |y - y64| <= c * u32 * sqrt(K) * (|A| . |B|)     u32 = 2^-24, c = 4, K = the full reduction length (however the
  kernel split it).  This is the probabilistic bound of Higham and Mary with enough margin for partial sums that are truncated rather
  than rounded to nearest at every step (wgmma's fp32 accumulation).  A link over it but under the deterministic K * u32 bound is
  reported with that ratio as well; the bound is not loosened.
* bf16 output: one more rounding, 2^-8 * |y64|.
* ReLU mask words written by a kernel: every bit must be y64 > 0 wherever |y64| exceeds the bound; inside it the bit may go either way,
  and that ambiguous fraction must stay below 1e-3 so that the check cannot become vacuous.
* element-wise kernels: the bound follows the fp32 operations the kernel performs (a few u32 per operation), plus the bf16 rounding.

Every comparator raises BoundError (an AssertionError) naming the link, and records the largest err / tol in a Report.
Everything here is plain torch and runs on the CPU as well as on the device.
"""
import math
from typing import List, Optional

import torch

U32 = 2.0 ** -24     # fp32 unit round-off
UBF = 2.0 ** -8      # bf16 unit round-off
U64 = 2.0 ** -53     # fp64 unit round-off
C_GEMM = 4.0
AMBIGUOUS_MAX = 1e-3


class BoundError(AssertionError):
    pass


def f64(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float64)


def f32r(x: float) -> float:
    """x rounded to fp32: the value a kernel receives for a float argument."""
    return float(torch.tensor(x, dtype=torch.float32))


class Report:
    """Per-link margins: the largest err / tol, the ambiguous-mask fraction, the excluded rows."""

    def __init__(self, title: str):
        self.title = title
        self.rows: List[tuple] = []

    def add(self, link: str, ratio: float, ambiguous: Optional[float] = None, excluded: Optional[str] = None) -> None:
        self.rows.append((link, ratio, ambiguous, excluded))

    def text(self) -> str:
        out = [f"== {self.title}"]
        for link, r, amb, exc in self.rows:
            s = f"  {link:<44s} err/tol {r:8.4f}"
            if amb is not None:
                s += f"  ambiguous {amb:.2e}"
            if exc is not None:
                s += f"  excluded {exc}"
            out.append(s)
        return "\n".join(out)


def _ratio(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor):
    err = (f64(got) - ref).abs()
    r = torch.where(tol > 0, err / torch.where(tol > 0, tol, torch.ones_like(tol)), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    if r.numel() == 0:
        return 0.0, None
    k = int(torch.argmax(r))
    return float(r.reshape(-1)[k]), k


def check(rep: Optional[Report], link: str, got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, det_tol: Optional[torch.Tensor] = None) -> float:
    """|got - ref| <= tol element-wise (ref, tol float64 of got's shape).  det_tol: the deterministic bound, reported on failure."""
    if got.shape != ref.shape:
        raise BoundError(f"{link}: shape {tuple(got.shape)} vs reference {tuple(ref.shape)}")
    r, k = _ratio(got, ref, tol)
    if rep is not None:
        rep.add(link, r)
    if not r < 1.0:
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(k), got.shape)) if k is not None else ()
        msg = (f"{link}: err/tol {r:.3f} at {idx}: got {float(got.reshape(-1)[k])!r}, reference {float(ref.reshape(-1)[k])!r}, "
               f"tol {float(tol.reshape(-1)[k]):.3e}")
        if det_tol is not None:
            rd, _ = _ratio(got, ref, det_tol)
            msg += f"; against the deterministic K*u32 bound: {rd:.3f}"
        raise BoundError(msg)
    return r


def check_exact(rep: Optional[Report], link: str, got: torch.Tensor, ref: torch.Tensor) -> None:
    bad = (f64(got) != f64(ref))
    if rep is not None:
        rep.add(link + " (exact)", float(bad.any()))
    if bad.any():
        k = int(torch.nonzero(bad.reshape(-1))[0])
        raise BoundError(f"{link}: {int(bad.sum())} elements differ; first at flat index {k}: {float(got.reshape(-1)[k])!r} "
                         f"vs {float(ref.reshape(-1)[k])!r}")


# ---------------------------------------------------------------------------------------------------------------------- GEMM links
def kernel_gemm(a, b, kblock=64, skip=None, dup_slice=None, slices=1):
    """CPU simulation of the GEMM kernels for the self-tests: fp32 accumulation of bf16 a [M, K] . b [K, N] block by block (each block
    product in fp32).  skip = (k-block, column slice): that k-block is left out of those columns.  slices / dup_slice: the reduction split
    into `slices` contiguous slices summed in order, slice `dup_slice` added twice."""
    a32, b32 = a.float(), b.float()
    K = a.shape[1]
    per = -(-K // slices)
    out = torch.zeros(a.shape[0], b.shape[1])
    for s in range(slices):
        part = torch.zeros_like(out)
        for k0 in range(s * per, min(K, (s + 1) * per), kblock):
            k1 = min(k0 + kblock, (s + 1) * per, K)
            blk = a32[:, k0:k1] @ b32[k0:k1]
            if skip is not None and skip[0] == k0 // kblock:
                blk[:, skip[1]] = 0.0
            part += blk
        out += part
        if s == dup_slice:
            out += part
    return out


class Gemm:
    """y64 = alpha * (A . B) [* gate] in float64 with its accumulation bound `acc` (before any output rounding)."""

    def __init__(self, a: torch.Tensor, b: torch.Tensor, alpha: float = 1.0, gate: Optional[torch.Tensor] = None,
                 bias: Optional[torch.Tensor] = None, c: float = C_GEMM):
        a, b = f64(a), f64(b)
        self.K = a.shape[1]
        y, ap = a @ b, a.abs() @ b.abs()
        if bias is not None:                      # fp32 epilogue add: one more term, one more rounding
            y, ap = y + f64(bias), ap + f64(bias).abs()
            self.K += 1
        self.acc = c * U32 * math.sqrt(self.K) * ap
        self.det = self.K * U32 * ap
        if bias is not None:
            self.acc = self.acc + U32 * y.abs()
            self.det = self.det + U32 * y.abs()
        if alpha != 1.0:                          # fp32 multiply of the accumulator
            y, self.acc, self.det = alpha * y, abs(alpha) * self.acc + U32 * abs(alpha) * y.abs(), abs(alpha) * self.det + U32 * abs(alpha) * y.abs()
        if gate is not None:                      # the kernel's own mask: gated elements are exactly zero
            g = gate.to(torch.float64)
            y, self.acc, self.det = y * g, self.acc * g, self.det * g
        self.y = y

    def tol(self, bf16: bool) -> torch.Tensor:
        return self.acc * (1 + UBF) + UBF * self.y.abs() if bf16 else self.acc

    def det_tol(self, bf16: bool) -> torch.Tensor:
        return self.det * (1 + UBF) + UBF * self.y.abs() if bf16 else self.det

    def check(self, rep: Optional[Report], link: str, got: torch.Tensor) -> float:
        bf16 = got.dtype == torch.bfloat16
        return check(rep, link, got, self.y, self.tol(bf16), self.det_tol(bf16))


def unpack_mask(words: torch.Tensor, n: int, m: int) -> torch.Tensor:
    """ReLU mask words int32 [ceil(n/32), >= m] (bit i of word (c, r) = column 32 c + i of row r) -> bool [m, n]."""
    w = words[:, :m].to(torch.int64) & 0xFFFFFFFF
    bits = (w[:, :, None] >> torch.arange(32, device=words.device)) & 1          # [W, m, 32]
    return bits.permute(1, 0, 2).reshape(m, -1)[:, :n].bool()


def pack_mask(bits: torch.Tensor) -> torch.Tensor:
    """Inverse of unpack_mask: bool [m, n] -> int32 [ceil(n/32), m]."""
    m, n = bits.shape
    wn = (n + 31) // 32
    full = torch.zeros(m, wn * 32, dtype=torch.int64, device=bits.device)
    full[:, :n] = bits.to(torch.int64)
    w = (full.view(m, wn, 32) << torch.arange(32, device=bits.device)).sum(-1)
    w = torch.where(w >= 2 ** 31, w - 2 ** 32, w)
    return w.T.contiguous().to(torch.int32)


def check_mask(rep: Optional[Report], link: str, words: torch.Tensor, g: Gemm, n: int, m: int) -> float:
    """Mask words a forward epilogue wrote for y = g.y: bit = y64 > 0 wherever |y64| exceeds the bound; bits past column n are 0."""
    bits = unpack_mask(words, ((n + 31) // 32) * 32, m)
    if bits[:, n:].any():
        raise BoundError(f"{link}: mask bits set past column {n}")
    bits = bits[:, :n]
    tol = g.tol(False)
    sure = g.y.abs() > tol
    wrong = sure & (bits != (g.y > 0))
    amb = float((~sure).double().mean())
    if rep is not None:
        rep.add(link, float(wrong.any()), ambiguous=amb)
    if wrong.any():
        r, c = (int(i) for i in torch.nonzero(wrong)[0])
        raise BoundError(f"{link}: {int(wrong.sum())} mask bits contradict the sign of y64, first at row {r} column {c} "
                         f"(y64 {float(g.y[r, c]):.3e}, bound {float(tol[r, c]):.3e})")
    if not amb < AMBIGUOUS_MAX:
        raise BoundError(f"{link}: {amb:.2e} of the mask bits lie within the bound (limit {AMBIGUOUS_MAX})")
    return amb


def sum_tol(terms_abs_sum: torch.Tensor, n: int, c: float = C_GEMM) -> torch.Tensor:
    """Bound of an fp32 sum of n terms whose magnitudes add up to terms_abs_sum (same model as the GEMM bound)."""
    return c * U32 * math.sqrt(max(n, 1)) * terms_abs_sum


# ---------------------------------------------------------------------------------------------------------------- element-wise links
def normalize_ref(x: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor, clamp: Optional[float] = 5.0):
    """clamp((x - mean) * rstd, +-clamp) -> bf16 (clamp None: unclamped): two fp32 roundings then one bf16 rounding."""
    x, m, r = f64(x), f64(mean), f64(rstd)
    y = (x - m) * r
    if clamp is not None:
        y = torch.clamp(y, -clamp, clamp)
    tol = UBF * y.abs() + 3 * U32 * (x.abs() + m.abs()) * r.abs() * (1 + UBF)
    return y, tol


def silu_tol(pre: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """Fast-math SiLU epilogue (ex2.approx / rcp.approx) on the bf16 pre-activation -- or, in a column group that reaches past N, on the
    fp32 accumulator, at most one bf16 rounding (2^-8 |pre|) away, |silu'| <= 1.1 -- and one bf16 rounding of the result."""
    shift = 1.1 * UBF * pre.abs() * (1 + UBF)
    return UBF * (s.abs() + shift) + shift + (8 + 2 * pre.abs()) * U32 * (s.abs() + pre.abs())


def silu64(z: torch.Tensor) -> torch.Tensor:
    return z * torch.sigmoid(z)


def silu_grad64(z: torch.Tensor) -> torch.Tensor:
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def silu_grad_err(z: torch.Tensor) -> torch.Tensor:
    """Bound of |act_grad_fast(z) - silu'(z)| for the dgrad gate (fast-math exp / divide, four fp32 operations)."""
    return (16 + 4 * z.abs()) * U32 * (1 + z.abs())


def silu_gated(g: "Gemm", pre: torch.Tensor):
    """A dgrad GEMM gated in its epilogue by silu'(pre) of the kernel's own bf16 pre-activation: (y64, accumulation bound before the
    bf16 output rounding).  Check with check(..., y, acc * (1 + UBF) + UBF * |y|)."""
    z = f64(pre)
    sg = silu_grad64(z)
    y = g.y * sg
    return y, g.acc * sg.abs() + g.y.abs() * silu_grad_err(z) + U32 * y.abs()


SILU_GRAD_ARGMAX = 2.3993572805154675      # z tanh(z / 2) = 2: where |silu'| peaks (1.09984 at +z*, 0.09984 at -z*)


def silu_grad_absmax(lo: torch.Tensor, hi: torch.Tensor) -> torch.Tensor:
    """max |silu'(z)| over [lo, hi]: the end points, and the two extrema of silu' where they lie inside."""
    m = torch.maximum(silu_grad64(lo).abs(), silu_grad64(hi).abs())
    for z in (SILU_GRAD_ARGMAX, -SILU_GRAD_ARGMAX):
        inside = (lo <= z) & (z <= hi)
        m = torch.where(inside, torch.maximum(m, silu_grad64(torch.tensor(z, dtype=torch.float64)).abs()), m)
    return m


def silu_gemm_tol(g: "Gemm") -> torch.Tensor:
    """SiLU in the forward epilogue, rounded to bf16 -- the eval path, where no pre-activation is stored.  The register epilogue applies
    it to the accumulator rounded to bf16 (fp32 only in a column group that reaches past N), so its argument lies within
    w = acc + one bf16 rounding of y: max |silu'| over [y - w, y + w] times w, the fast-math SiLU evaluation (as in silu_tol), one bf16
    rounding of the result."""
    w = g.acc * (1 + UBF) + UBF * g.y.abs()
    z = g.y.abs() + w
    s = silu64(g.y)
    shift = silu_grad_absmax(g.y - w, g.y + w) * w + (8 + 2 * z) * U32 * (s.abs() + z)
    return shift + UBF * (s.abs() + shift)


def gaussian_sample_ref(mu: torch.Tensor, eps: torch.Tensor, logstd: torch.Tensor):
    """pulse_gaussian_sample on the kernel's own mu: actions = mu + exp(logstd) eps and neglogp = 0.5 sum z^2 + 0.5 log(2 pi) A +
    sum logstd with z = (a - mu) / sigma, float64, with the bounds of the fp32 kernel (expf, the product and the sum for a; for z the
    cancellation a - mu, the quotient; then the per-lane and warp sums of A terms and the fp32 constant 0.5f * log(2 pi)f * A)."""
    mu, eps, ls = f64(mu), f64(eps), f64(logstd)
    A = mu.shape[1]
    sg = torch.exp(ls)
    a = mu + sg * eps
    tol_a = U32 * a.abs() + 3 * U32 * (sg * eps).abs()
    dz = (tol_a + U32 * (a - mu).abs()) / sg + 3 * U32 * eps.abs()
    z2 = eps * eps
    nlp = 0.5 * z2.sum(-1) + 0.5 * math.log(2 * math.pi) * A + ls.sum()
    c32 = 0.5 * f32r(1.8378770664093453) * A
    tol_n = (0.5 * (2 * eps.abs() * dz + dz * dz + U32 * z2).sum(-1) + 0.5 * A * U32 * z2.sum(-1) + A * U32 * ls.abs().sum()
             + abs(c32 - 0.5 * math.log(2 * math.pi) * A) + 2 * U32 * c32 + 2 * U32 * (nlp.abs() + c32 + ls.abs().sum()))
    return a, tol_a, nlp, tol_n


def value_unnorm_ref(y: torch.Tensor, mean: torch.Tensor, var: torch.Tensor, eps: float, terminate: Optional[torch.Tensor] = None):
    """value_unnorm.cuh on the kernel's own normalised value y: clamp(y, +-5) * sqrt(var.float() + eps) + mean.float() [* (1 - terminate)],
    float64.  fp32: the add under the root, the root (half the relative error of its argument, plus its own rounding), the product and
    the sum -- one u32 each; the terminate factor is exactly 0 or 1."""
    c = torch.clamp(f64(y), -5.0, 5.0)
    m = float(mean.reshape(-1)[0].float())
    sd = math.sqrt(float(var.reshape(-1)[0].float()) + f32r(eps))
    v = c * sd + m
    tol = 3 * U32 * (c * sd).abs() + U32 * v.abs()
    if terminate is not None:
        keep = 1.0 - f64(terminate)
        v, tol = v * keep, tol * keep
    return v, tol


def pd_targets_exact(actions: torch.Tensor, offset: torch.Tensor, scale: torch.Tensor, freeze: Optional[torch.Tensor] = None):
    """Humanoid._action_to_pd_targets as the kernels round it: fp32(offset + fp32(scale * a)), two separate roundings -- exact, so the
    kernel's targets must match bit for bit (frozen dofs: exactly 0)."""
    t = offset.float()[None, :] + scale.float()[None, :] * actions.float()
    if freeze is not None:
        t = torch.where(freeze.bool()[None, :], torch.zeros_like(t), t)
    return t


def policy_post_ref(mu, eps, logstd, eps_tol=None, value=None, value_mean=None, value_var=None, value_eps=1e-5):
    """policy_post_kernel on the kernel's own head output mu: actions and neglogp through gaussian_sample_ref (same fp32 operations),
    the de-normalised value (value_unnorm_ref).  eps_tol: the draws are the fp64 regeneration of the kernel's Philox noise
    (philox_normals_ref), off by at most eps_tol -- it widens the action bound by sigma * eps_tol and neglogp's by sum (|eps| + eps_tol/2)
    eps_tol.  The PD targets are exact: pd_targets_exact on the kernel's actions.  Returns {name: (value, tol)} in float64."""
    a, tol_a, nlp, tol_n = gaussian_sample_ref(mu, eps, logstd)
    if eps_tol is not None:
        et = f64(eps_tol)
        tol_a = tol_a + torch.exp(f64(logstd)) * et
        tol_n = tol_n + ((f64(eps).abs() + 0.5 * et) * et).sum(-1)
    out = {"actions": (a, tol_a), "neglogp": (nlp, tol_n)}
    if value is not None:
        out["values"] = value_unnorm_ref(value, value_mean, value_var, value_eps) if value_mean is not None else (f64(value), torch.zeros_like(f64(value)))
    return out


def latent_post_ref(mu, eps, logstd, prior_mu, actions, eps_tol=None, value=None, value_mean=None, value_var=None, value_eps=1e-5):
    """latent_post_kernel on the kernel's own head mu and prior mean: policy_post_ref's actions, neglogp and value (the same draws and
    arithmetic), and the decoder's latent z = bf16(fp32(prior_mu + a)) from the kernel's own actions -- two correctly rounded
    operations, so "z" is exact (bf16)."""
    out = policy_post_ref(mu, eps, logstd, eps_tol=eps_tol, value=value, value_mean=value_mean, value_var=value_var, value_eps=value_eps)
    out["z"] = (prior_mu.float() + actions.float()).to(torch.bfloat16)
    return out


def philox_normals_ref(seed: int, index, offset):
    """Box-Muller (philox.cuh) in float64 on the Philox4x32-10 blocks (seed, index, offset) regenerated on the host: returns
    (n0, n1, tol0, tol1), the normals of words x / y, float64 tensors of index's shape.

    The kernel forms u1 = (x >> 8 + 1) 2^-24 and u2 = (y >> 8) 2^-24 exactly, then r = sqrtf(-2 __logf(u1)) and __sincosf(2 pi_f32 u2).
    __logf is lg2.approx.f32 times ln 2 (one fp32 multiply).  The error figures below are the ones the CUDA C++ programming guide gives
    for __logf and __sinf / __cosf (2^-21.41 absolute on [0.5, 2], 3 ulp elsewhere; 2^-21.41 absolute on [-pi, pi]) and the PTX ISA
    manual for lg2.approx.f32 and sin.approx / cos.approx.f32; the looser figure is used wherever the two differ.  The logarithm:
    E_log = max(2^-21.41, 3 ulp of |ln u1|) plus the multiply by ln 2; r then carries sqrt(r^2 + 2 E_log) - r (finite as r -> 0,
    where u1 -> 1) plus the rounding of the root.  The sine and cosine: 2^-20.5 over [-pi, pi].  The argument 2 pi u2 covers [0, 2 pi),
    and neither document gives a figure on (pi, 2 pi); there this bound takes 2^-20, an assumption (twice the [-pi, pi] figure, for the
    range reduction's extra rounding at 2 pi), which no test isolates: the GPU checks confirm only that the combined bound holds.  The
    argument itself is off by one rounding of the product (the reference uses the same fp32 constant 2 pi_f32).
    All of it stays near 1e-6 for most draws (below 1e-4 as u1 -> 1), far below the O(1) difference of a draw from another Philox
    block."""
    import numpy as np
    from tests.philox_ref import philox4x32_10
    x, y, _, _ = philox4x32_10(seed, index, offset)
    u1 = ((x >> np.uint64(8)).astype(np.float64) + 1.0) / 16777216.0
    u2 = (y >> np.uint64(8)).astype(np.float64) / 16777216.0
    ln = np.log(u1)
    r = np.sqrt(-2.0 * ln)
    two_pi_f32 = float(np.float32(2 * math.pi))
    arg = two_pi_f32 * u2
    c, s = np.cos(arg), np.sin(arg)
    e_log = np.maximum(2.0 ** -21.41, 3 * 2 * U32 * np.abs(ln)) + U32 * np.abs(ln)        # + the fp32 multiply by ln 2
    dr = 2 * e_log / (np.sqrt(r * r + 2 * e_log) + r) + U32 * r                                 # -2 ln exact; sqrtf rounds once
    e_trig = np.where(arg <= math.pi, 2.0 ** -20.5, 2.0 ** -20) + U32 * arg       # the reference uses 2 pi_f32: one rounding of the product
    n0, n1 = r * c, r * s
    t0 = dr * np.abs(c) + r * e_trig + U32 * np.abs(n0) + dr * e_trig
    t1 = dr * np.abs(s) + r * e_trig + U32 * np.abs(n1) + dr * e_trig
    to = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64))
    return to(n0), to(n1), to(t0), to(t1)


def philox_pair_normals(seed: int, rows: int, width: int, offset: int, stride: int = 64):
    """The normals of a [rows, width] draw laid out as the kernels lay it: columns (2p, 2p + 1) are the Box-Muller pair of block
    (seed, row * stride + p, offset).  Returns (n, tol) float64 [rows, width]."""
    import numpy as np
    pairs = (width + 1) // 2
    idx = (np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(stride) + np.arange(pairs, dtype=np.uint64)[None, :]).reshape(-1)
    n0, n1, t0, t1 = philox_normals_ref(seed, idx, offset)
    n = torch.stack([n0, n1], -1).reshape(rows, 2 * pairs)[:, :width]
    t = torch.stack([t0, t1], -1).reshape(rows, 2 * pairs)[:, :width]
    return n, t


def pnn_compose_ref(w: torch.Tensor, acts: torch.Tensor, act: Optional[str]):
    """pnn_compose_kernel on the kernel's own composer head w [M, K] and primitive outputs acts [K, M, A]: sum_k act(w_k) a_k, float64.
    fp32: act(w) (SiLU as w / (1 + expf(-w)): expf, the add, the quotient -- 4 u32 of |silu| plus expf's 2 ulp carried through), then
    K fused multiply-adds -- one rounding each, bounded by K u32 sum |act(w_k) a_k|."""
    w64, a64 = f64(w), f64(acts)
    if act == "silu":
        g = silu64(w64)
        eg = 6 * U32 * (g.abs() + (w64 * torch.sigmoid(w64) * (1 - torch.sigmoid(w64))).abs())
    elif act == "relu":
        g, eg = torch.relu(w64), torch.zeros_like(w64)
    else:
        g, eg = w64, torch.zeros_like(w64)
    K = w.shape[1]
    terms = g.T[:, :, None] * a64                       # [K, M, A]
    y = terms.sum(0)
    tol = K * U32 * terms.abs().sum(0) + (eg.T[:, :, None] * a64.abs()).sum(0) + U32 * y.abs()
    return y, tol


def reparam_ref(head: torch.Tensor, noise: torch.Tensor, mode: str, latent: int, clamp: bool = True, lo: float = -5.0, hi: float = 2.0,
                noise_tol: Optional[torch.Tensor] = None):
    """vae_reparam_kernel / vae_reparam_philox_kernel on the kernel's own head [M, >= 2 latent], rounded to bf16, float64:
    'sample'   z = mu + exp(0.5 clamp(logvar)) eps   (0.5 lv exact; expf within 2 ulp, 4 u32; the product and the sum, one rounding each:
               5 u32 |sigma eps| + u32 |z| covers them whether or not the compiler contracts them into one fma),
    'mean'     z = mu                                 (exact: the bf16 rounding of mu),
    'residual' z = mu + eps                           (one rounding).
    noise_tol: eps is the fp64 regeneration of the kernel's draws (philox_normals_ref), off by at most noise_tol."""
    h = f64(head)
    mu = h[:, :latent]
    if mode == "mean":
        return mu, UBF * mu.abs()
    e = f64(noise)[:, :latent]
    if mode == "residual":
        z = mu + e
        tol = U32 * z.abs()
        if noise_tol is not None:
            tol = tol + f64(noise_tol)
    else:
        lv = h[:, latent:2 * latent]
        if clamp:
            lv = torch.clamp(lv, lo, hi)
        sg = torch.exp(0.5 * lv)
        z = mu + sg * e
        tol = U32 * z.abs() + 5 * U32 * (sg * e).abs()
        if noise_tol is not None:
            tol = tol + sg * f64(noise_tol)
    return z, UBF * z.abs() + (1 + UBF) * tol


def gae_ref(rewards, values, next_values, dones, gamma: float, tau: float):
    """gae_kernel in float64 on fp32 time-major [T, N] inputs: delta = r + g V' - V, last = delta + (g tau)(1 - d) last, ret = last + V,
    with the kernel's fp32 constant g tau = fp32(fp32(g) fp32(tau)) (an exact product, rounded once).  The bound is carried backwards
    step by step: delta costs three roundings (u32 |g V'|, u32 |r + g V'|, u32 |delta|); each step adds delta's error, the rounding of
    the product (u32 |c (1-d) last|) and of the sum (u32 |last|) to the error of the step after it, shrunk by c (1 - d).  So it scales
    with |r|, |V| and |V'| and grows along t only as far as the discounting lets it.  Returns (adv, tol_adv, ret, tol_ret) time-major."""
    r, v, nv, d = f64(rewards), f64(values), f64(next_values), f64(dones)
    g = f32r(gamma)
    c = f32r(g * f32r(tau))
    T = r.shape[0]
    adv, ret = torch.zeros_like(r), torch.zeros_like(r)
    ta, tr = torch.zeros_like(r), torch.zeros_like(r)
    last, err = torch.zeros_like(r[0]), torch.zeros_like(r[0])
    for t in range(T - 1, -1, -1):
        gv = g * nv[t]
        s = r[t] + gv
        delta = s - v[t]
        e_delta = U32 * (gv.abs() + s.abs() + delta.abs())
        carry = c * (1.0 - d[t]) * last                 # c (1 - d) is exact in fp32: d is 0 or 1
        e_prod = c * (1.0 - d[t]) * err + U32 * (carry.abs() + c * err)
        last = delta + carry
        err = e_delta + e_prod + U32 * (last.abs() + e_delta + e_prod)
        adv[t], ta[t] = last, err
        ret[t] = last + v[t]
        tr[t] = err + U32 * (ret[t].abs() + err)
    return adv, ta, ret, tr


def adv_normalize_ref(adv: torch.Tensor):
    """normalize_adv_kernel on the kernel's own fp32 advantages a (flat [n]): (a - fp32(mean)) / (fp32(sqrt(unbiased var)) + 1e-8f),
    float64.  The fp64 sums are exact to n u64 of sum |a| and sum a^2 (any order); mean and variance follow within a few u64 per
    operation, which may move fp32(mean) / fp32(sqrt var) by one rounding each: u32 |mean| / den and u32 |y| (twice: the root and the
    +1e-8f add).  Then the fp32 difference (u32 |a - mean| / den) and the quotient (u32 |y|)."""
    a = f64(adv).reshape(-1)
    n = a.numel()
    s, q = a.sum(), (a * a).sum()
    mean = s / n
    var = torch.clamp((q - n * mean * mean) / (n - 1), min=0.0)
    e_mean = float(U64 * a.abs().sum() + U64 * mean.abs())
    e_var = float((n * U64 * q + 2 * n * mean.abs() * e_mean + 4 * U64 * (q + n * mean * mean)) / (n - 1))
    sd = math.sqrt(float(var))
    m32 = f32r(float(mean))
    den = f32r(f32r(sd) + f32r(1e-8))
    y = (a - m32) / den
    e_m = e_mean + 2 * U32 * abs(m32)                           # the kernel's fp32(mean) may round the other way
    e_den = (e_var / (2 * sd) if sd > 0 else math.sqrt(e_var)) + 4 * U32 * den
    tol = (U32 * (a - m32).abs() + e_m) / den + y.abs() * (e_den / den + U32)
    return y, tol


def ppo_loss_ref(mu, value, actions, old_nlp, adv, ret, logstd, old_mu=None, e_clip=0.2, critic_coef=5.0, bounds_coef=10.0):
    """pulse_ppo_loss on the kernel's own mu / value: float64 autograd of the oracle's ppo_total_loss (dmu, dv), the per-row statistics
    and the bounds of the fp32 kernel.  Rows whose branch decision lies within rounding of its threshold are flagged `ambiguous`."""
    from oracle import pulse_oracle as po
    M, A = mu.shape
    mu64 = f64(mu).requires_grad_(True)
    v64 = f64(value).reshape(M).requires_grad_(True)
    act, onl, adv64, ret64, ls = f64(actions), f64(old_nlp), f64(adv), f64(ret), f64(logstd)
    r = po.ppo_total_loss(mu64, v64, onl, adv64, ret64, act, ls, e_clip=e_clip, critic_coef=critic_coef, bounds_coef=bounds_coef)
    dmu, dv = torch.autograd.grad(r["loss"], (mu64, v64))
    with torch.no_grad():
        sg = torch.exp(ls)
        z = (act - mu64) / sg
        nlp = r["neglogp"]
        d = onl - nlp
        ratio = torch.exp(d)
        nlp_mag = 0.5 * (z * z).sum(-1) + 0.5 * math.log(2 * math.pi) * A + ls.abs().sum()
        ratio_rel = 16 * U32 * nlp_mag + U32 * d.abs() + 4 * U32            # error of nlp, of the difference, of expf
        lo, hi = 1.0 - f32r(e_clip), 1.0 + f32r(e_clip)
        win = 2 * ratio * ratio_rel
        ambiguous = ((ratio - lo).abs() <= win) | ((ratio - hi).abs() <= win)
        mu_d = mu64.detach()
        bnd_edge = ((mu_d.abs() - 1.0).abs() <= 4 * U32 * mu_d.abs()).any(-1)     # |mu| ~ 1: the bound loss's kink
        ambiguous = ambiguous | bnd_edge
        rc = torch.clamp(ratio, lo, hi)
        active = (-adv64 * ratio) >= (-adv64 * rc)
        dnlp_dmu = -(act - mu_d) / (sg * sg)
        ta = torch.where(active, adv64 * ratio, torch.zeros_like(ratio))[:, None] * dnlp_dmu / M
        hi_t, lo_t = torch.clamp_min(mu_d - 1.0, 0.0), torch.clamp_max(mu_d + 1.0, 0.0)
        tb = bounds_coef * 2.0 * (hi_t + lo_t) / M
        tol_mu = UBF * dmu.abs() + (1 + UBF) * ((ratio_rel[:, None] + 8 * U32) * ta.abs() + 8 * U32 * tb.abs())
        tol_v = UBF * dv.abs() + 6 * U32 * (critic_coef * 2.0 * (ret64.abs() + v64.detach().abs()) / M)
        a_loss = torch.maximum(-adv64 * ratio, -adv64 * rc)
        c_loss = (ret64 - v64.detach()) ** 2
        b_loss = (hi_t ** 2 + lo_t ** 2).sum(-1)
        stats = [a_loss.sum(), c_loss.sum(), b_loss.sum(), None, ((ratio - 1.0).abs() > f32r(e_clip)).double().sum(), nlp.sum()]
        stats_tol = [(adv64.abs() * ratio * (ratio_rel + 4 * U32)).sum(), (8 * U32 * ((ret64.abs() + v64.detach().abs()) ** 2)).sum(),
                     (8 * U32 * (hi_t.abs() + lo_t.abs() + 1) ** 2).sum(), None, float(ambiguous.sum()), (16 * U32 * nlp_mag).sum()]
        if old_mu is not None:
            sg2 = sg * sg
            dd = f64(old_mu) - mu_d
            frac = (sg2 + dd * dd) / (2.0 * (sg2 + f32r(1e-5)))
            stats[3] = (math.log(1.0 + f32r(1e-5)) + frac - 0.5).sum()
            # per term: expf(logstd), the squares, the difference old_mu - mu and the quotient, a few u32 of (1 + frac) each
            stats_tol[3] = (16 * U32 * (1.5 + frac + dd.abs() * (f64(old_mu).abs() + mu_d.abs()) / sg2)).sum()
    return {"dmu": dmu, "dv": dv, "tol_mu": tol_mu, "tol_v": tol_v, "ambiguous": ambiguous, "stats": stats, "stats_tol": stats_tol,
            "ratio": ratio, "active": active}


def disc_loss_ref(logits: torch.Tensor, n_agent: int, scale: float):
    """pulse_disc_loss: dlogit = 0.5 * scale * d(mean BCE)/dl per batch (agent rows target 0, demo rows target 1), the statistics."""
    l = f64(logits).reshape(-1)
    n = l.shape[0]
    n_demo = n - n_agent
    sg = torch.sigmoid(l)
    agent = torch.arange(n, device=l.device) < n_agent
    g = torch.where(agent, 0.5 * scale * sg / n_agent, 0.5 * scale * (sg - 1.0) / n_demo)
    cnt = torch.where(agent, torch.full_like(l, float(n_agent)), torch.full_like(l, float(n_demo)))
    tol = UBF * g.abs() + 8 * U32 * 0.5 * scale * (sg + 1.0) / cnt
    sp = torch.nn.functional.softplus(l)
    spm = torch.nn.functional.softplus(-l)
    stats = [sp[agent].sum(), spm[~agent].sum(), (l[agent] < 0).double().sum(), (l[~agent] > 0).double().sum()]
    stats_tol = [(8 * U32 * (sp[agent] + l[agent].abs() + 1)).sum(), (8 * U32 * (spm[~agent] + l[~agent].abs() + 1)).sum(), 0.0, 0.0]
    return g, tol, stats, stats_tol


def adam_ref(p, g, m, v, step: int, *, lr: float, max_norm: float, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8,
             sumsq_rel: float = 16 * U32):
    """clip_grad_norm_(max_norm) + torch.optim.Adam step number step + 1 in float64 on fp32 state, with the bounds of the fp32 kernel.
    The constants are the fp32 values the kernel receives.  Returns (p, m, v, tol_p, tol_m, tol_v, clipped, norm_margin)."""
    lr, b1, b2, eps = f32r(lr), f32r(b1), f32r(b2), f32r(eps)
    p, g, m, v = f64(p), f64(g), f64(m), f64(v)
    t = step + 1
    norm = float(torch.sqrt((g * g).sum()))
    scale, clipped, margin = 1.0, False, math.inf
    if max_norm and max_norm > 0:
        mn = f32r(max_norm)
        scale = min(1.0, mn / (norm + f32r(1e-6)))
        clipped = scale < 1.0
        margin = abs(norm / mn - 1.0)
    gs = g * scale
    rel_g = (sumsq_rel + 4 * U32 if clipped else 0.0) + U32
    dg = gs.abs() * rel_g
    m1 = b1 * m + (1 - b1) * gs
    v1 = b2 * v + (1 - b2) * gs * gs
    dm = 2 * U32 * (b1 * m.abs() + (1 - b1) * gs.abs()) + (1 - b1) * dg + U32 * m1.abs()
    dv = 3 * U32 * (b2 * v + (1 - b2) * gs * gs) + (1 - b2) * 2 * gs.abs() * dg
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    rel_bc1 = 8 * U32 * b1 ** t / bc1 + U32          # powf: a few ulp of b^t, then the subtraction
    rel_bc2 = 8 * U32 * b2 ** t / bc2 + U32
    s = torch.sqrt(v1) / math.sqrt(bc2)
    den = s + eps
    st = (lr / bc1) * m1 / den
    p1 = p - st
    rel_v = torch.where(v1 > 0, dv / torch.where(v1 > 0, v1, torch.ones_like(v1)), torch.zeros_like(v1))
    dden = s * (0.5 * rel_v + 0.5 * rel_bc2 + 4 * U32) + U32 * den
    dst = st.abs() * (rel_bc1 + 4 * U32) + (lr / bc1) * (dm / den + m1.abs() * dden / (den * den))
    dp = U32 * (p1.abs() + p.abs()) + dst
    return p1, m1, v1, dp, dm, dv, clipped, margin


def latent_loss_tol(enc, pri, noise, dz, progress, E: int, T: int, kld_coef: float, ar1_coef: float, clamp=(-5.0, 2.0), phi: float = 0.99):
    """Bounds of pulse_vae_latent_loss's head gradients (d_enc, d_prior) from the fp32 operations it performs, float64 [M, 2E] each."""
    enc, pri, noise, dz = f64(enc), f64(pri), f64(noise), f64(dz)
    M = enc.shape[0]
    qm, pm = enc[:, :E], pri[:, :E]
    qv, pv = torch.clamp(enc[:, E:], *clamp), torch.clamp(pri[:, E:], *clamp)
    kc = kld_coef / M
    ipv, ratio, dm = torch.exp(-pv), torch.exp(qv - pv), qm - pm
    ddm = U32 * (qm.abs() + pm.abs())
    dratio = ratio * (U32 * (qv - pv).abs() + 3 * U32)
    t_qm = kc * ipv * (ddm + 4 * U32 * dm.abs()) + U32 * dz.abs()
    t_qv = kc * 0.5 * (dratio + U32 * (ratio + 1)) + 6 * U32 * (dz * 0.5 * torch.exp(0.5 * qv) * noise).abs()
    t_pv = kc * 0.5 * (dratio + 2 * dm.abs() * ddm * ipv + 6 * U32 * dm * dm * ipv + U32 * (1 + ratio + dm * dm * ipv))
    t_pm = t_qm - U32 * dz.abs()
    if ar1_coef:
        pairs = (M // T) * (T - 1)
        c = ar1_coef / pairs
        prog = progress.to(torch.int64)
        t = torch.arange(M, device=enc.device) % T
        keep = torch.zeros(M, dtype=torch.bool, device=enc.device)        # pair (r - 1, r)
        keep[1:] = ((prog[1:] - prog[:-1]) == 1) & ~((prog[1:] <= 2) | (prog[:-1] <= 2)) & (t[1:] > 0)
        e = torch.zeros_like(qm)
        e[1:] = qm[1:] - f32r(phi) * qm[:-1]
        de = torch.zeros_like(qm)
        de[1:] = U32 * (qm[1:].abs() + 2 * qm[:-1].abs())
        nrm = e.norm(dim=-1, keepdim=True)
        dn = (e.abs() * de).sum(-1, keepdim=True) / nrm.clamp_min(1e-300) + (E + 4) * U32 * nrm
        term = c * (de / nrm.clamp_min(1e-300) + e.abs() * dn / nrm.clamp_min(1e-300) ** 2 + 4 * U32 * e.abs() / nrm.clamp_min(1e-300))
        term = torch.where(keep[:, None] & (nrm > 0), term, torch.zeros_like(term))
        t_qm = t_qm + term
        t_qm[:-1] = t_qm[:-1] + f32r(phi) * term[1:]
    return torch.cat([t_qm, t_qv], 1), torch.cat([t_pm, t_pv], 1)
