"""pulse_gemm_bf16 cell by cell against float64: operand families, guard-banded buffers, the dispatch model and the cell table.

One GEMM call lands in one of many kernels -- operand layout x epilogue mode x ring depth x tile width x output path (gemm_wgmma.cu,
launch_gemm / epilogue_maps).  A Case names the request (shape, layout, epilogue, strides); `predict` is the host dispatch written out, so
a test can assert that the launch took the kernel the case was written for (pulse_gemm_last_launch), and CELLS lists the cells the cases
must reach.

Two operand families per case:
* exact -- small integers laid out as position-dependent patterns, integer bias, power-of-two alpha.  Every product is exact in fp32 and
  every partial sum stays below 2^22, so the fp32 result is exact in any summation order or split: fp32 outputs, weight-gradient sums,
  slabs and column sums must equal the fp64 value, bf16 outputs its round-to-nearest-even, mask bits y > 0 (y == 0 included).  Where a
  case asks for the sum of squares, its operands are small and sparse enough that every fp32 partial the kernel can form (at most one
  warp's 32 rows x 128 columns) is exact too (`sumsq_exact`).  SiLU is not exact in either family: it keeps its rounding bound.
* bounded -- random normal operands, held to the fp64_ref.Gemm bound (plus one bf16 rounding), SiLU to silu_gemm_tol / silu_gated.
Alpha is a power of two, folded into A for the bounded reference (alpha * A . B + bias is what the kernel computes; fp64_ref.Gemm would
scale the bias too).

Every output is a window inside a larger buffer whose rest holds sentinels (NaN fp32, a fixed bf16 pattern, 0x5A5A5A5A mask words):
after the call everything outside the window must be unchanged bit for bit.  Operand padding (columns past the contiguous extent, rows
past the other one) holds bf16 NaN, so a load outside a tensor map's extent poisons the output instead of reading zeros by luck.
Plain torch: runs on the CPU and on the device.
"""
import math
import random
from dataclasses import dataclass, replace
from typing import Dict, List, Optional

import torch

from tests.fp64_ref import (BoundError, Gemm, U32, UBF, Report, check, check_exact, check_mask, f64, silu64, silu_gated,
                            silu_gemm_tol, sum_tol, unpack_mask)

MODE_GENERIC, MODE_FWD, MODE_DGRAD, MODE_WGRAD, MODE_DGRAD_VEC = 0, 1, 2, 3, 4
MODE_NAMES = {MODE_GENERIC: "generic", MODE_FWD: "fwd", MODE_DGRAD: "dgrad", MODE_WGRAD: "wgrad", MODE_DGRAD_VEC: "dgrad_vec"}
TMA_NAMES = {0: "staged", 1: "tma", 2: "reg_f32"}
BM, BK, NARROW, WIDE, WIDE_MIN_KB = 128, 64, 128, 256, 4
H100_SMS = 132
BF16_SENTINEL = 0x7FA5          # a NaN payload no rounding produces
MASK_SENTINEL = 0x5A5A5A5A
BF16_NAN = 0x7FC0
VARIANTS = {"default": {}, "stages4": {"PULSE_GEMM_STAGES": "4"}, "bn128": {"PULSE_GEMM_BN": "128"}}


def _ceil(a: int, b: int) -> int:
    return -(-a // b)


def num_splits(k: int, split_k: int) -> int:
    """pulse_gemm_num_splits: every slab gets at least one k-block."""
    nkb = _ceil(k, BK)
    s = max(1, min(split_k, nkb))
    per = _ceil(nkb, s)
    return _ceil(nkb, per)


def kb_per_split(k: int, split_k: int) -> int:
    return _ceil(_ceil(k, BK), num_splits(k, split_k))


def slab_range(k: int, split_k: int, z: int):
    """k range [k0, k1) of split-K slab z."""
    per = kb_per_split(k, split_k) * BK
    return z * per, min(k, (z + 1) * per)


# ------------------------------------------------------------------------------------------------------------------------------ cases
@dataclass(frozen=True)
class Case:
    name: str
    M: int
    N: int
    K: int
    a_mn: bool = False
    b_mn: bool = False
    out: bool = True              # bf16 output
    f32: str = ""                 # fp32 output: "" | "plain" | "slabs" | "accum" (raw accumulate) | "dense" (dense.gemm accumulate + split)
    out_t: bool = False
    preact: bool = False
    bias: bool = False
    act: str = "none"             # none | relu | silu
    alpha: float = 1.0            # a power of two
    gate: str = ""                # "" | relu (bf16 saved output) | silu (bf16 pre-activation) | bits (mask words)
    colsum: bool = False
    sumsq: bool = False
    relu_mask: bool = False
    split_k: int = 1
    ldo_odd: bool = False         # bf16 output rows (out, preact, out_t) with ld % 8 != 0
    ldf_odd: bool = False         # fp32 output rows with ldf % 4 != 0
    f32_shift: bool = False       # fp32 output base 4 bytes past a 16-byte boundary
    ldg_odd: bool = False         # gate rows with ldg % 8 != 0
    cell: str = ""                # the CELLS row the default dispatch on an H100 must reach ("" = none in particular)

    @property
    def layout(self) -> str:
        return ("amn" if self.a_mn else "ak") + "_" + ("bmn" if self.b_mn else "bk")


def epilogue_mode(c: Case) -> int:
    """gemm_wgmma.cu epilogue_mode: the smallest specialisation that covers the request."""
    want_fwd = c.bias or c.act != "none" or c.preact or c.out_t or c.relu_mask
    want_dgrad = bool(c.gate) or c.colsum or c.sumsq
    accum = c.f32 == "accum"
    if not want_dgrad and not accum:
        return MODE_FWD
    if not want_fwd and not accum:
        return MODE_DGRAD_VEC if c.gate == "silu" else MODE_DGRAD
    if not want_fwd and not want_dgrad and not c.out and c.alpha == 1.0:
        return MODE_WGRAD
    return MODE_GENERIC


def tile_n(m: int, n: int, kbpi: int, splits: int, sms: int) -> int:
    """gemm_tile_n: the wide tile where it does not cost a round."""
    if n < WIDE or kbpi < WIDE_MIN_KB or sms < 1:
        return NARROW
    tm = _ceil(m, BM)
    rn = _ceil(tm * _ceil(n, NARROW) * splits, sms)
    rw = _ceil(tm * _ceil(n, WIDE) * splits, sms)
    return WIDE if 2 * rw <= rn else NARROW


def predict(c: Case, sms: int, variant: str = "default") -> Dict[str, int]:
    """The kernel the host dispatch picks for c (launch_gemm, epilogue_maps, ring_stages, gemm_tile_n), as pulse_gemm_last_launch
    reports it."""
    stages4, bn128 = variant == "stages4", variant == "bn128"
    mode = epilogue_mode(c) if c.f32 != "dense" else MODE_FWD
    ns = num_splits(c.K, c.split_k)
    f32_ok = c.f32 == "dense" or (not c.ldf_odd and not c.f32_shift)      # dense allocates its own aligned slabs
    tma = 0
    if mode == MODE_WGRAD:
        tma = 1 if f32_ok and c.N % 4 == 0 else 0
    elif (mode == MODE_FWD and c.f32 in ("plain", "slabs", "dense") and not (c.out or c.out_t or c.preact or c.relu_mask or c.bias)
          and c.act == "none" and c.alpha == 1.0 and c.N % 4 == 0 and f32_ok):
        tma = 2
    elif (mode in (MODE_FWD, MODE_DGRAD) and c.N % 8 == 0 and c.out and not c.f32 and not c.out_t and c.gate in ("", "bits")
          and not c.colsum and not c.ldo_odd):
        tma = 1
    S, BN = 4, NARROW
    if mode in (MODE_FWD, MODE_DGRAD):
        s = 4 if (tma == 0 or stages4) else (5 if c.preact else 6)
        if s == 4 and tma == 2:
            tma = 0
        if (not c.a_mn and s != 4 and tma == 1 and not c.preact and not bn128
                and tile_n(c.M, c.N, kb_per_split(c.K, c.split_k), ns, sms) == WIDE):
            BN = WIDE
        elif s == 6 or (s == 5 and mode == MODE_FWD):
            S = s
    total = _ceil(c.N, BN) * _ceil(c.M, BM) * ns
    return {"mode": mode, "stages": S, "tile_n": BN, "tma_out": tma, "splits": ns, "grid": min(total, sms)}


def cell_name(c: Case, L: Dict[str, int]) -> str:
    return f"{c.layout}/{MODE_NAMES[L['mode']]}/S{L['stages']}/BN{L['tile_n']}/{TMA_NAMES[L['tma_out']]}"


def _reg(L, mode, S=None, BN=NARROW, tma=1):
    return L["mode"] == mode and L["tma_out"] == tma and L["tile_n"] == BN and (S is None or L["stages"] == S)


def _staged(L, mode):
    return L["mode"] == mode and L["tma_out"] == 0 and L["stages"] == 4 and L["tile_n"] == NARROW


# The cells the suite must reach: (id, predicate on (case, launch, variant)).  A launch counts for a row only once its case has passed.
CELLS = [
    ("fwd reg bf16 S6 BN128 + bias", lambda c, L, v: _reg(L, MODE_FWD, 6) and c.bias),
    ("fwd reg bf16 S6 BN128 + relu + mask words", lambda c, L, v: _reg(L, MODE_FWD, 6) and c.act == "relu" and c.relu_mask),
    ("fwd reg bf16 S6 BN128 + silu", lambda c, L, v: _reg(L, MODE_FWD, 6) and c.act == "silu"),
    ("fwd reg bf16 + preact S5", lambda c, L, v: _reg(L, MODE_FWD, 5) and c.preact),
    ("fwd reg bf16 BN256, B K-major", lambda c, L, v: _reg(L, MODE_FWD, 4, WIDE) and not c.b_mn),
    ("fwd reg bf16 BN256, B MN-major", lambda c, L, v: _reg(L, MODE_FWD, 4, WIDE) and c.b_mn),
    ("fwd reg bf16 under PULSE_GEMM_STAGES=4", lambda c, L, v: v == "stages4" and _reg(L, MODE_FWD, 4) and c.out),
    ("fwd reg fp32 slabs, split 1", lambda c, L, v: _reg(L, MODE_FWD, 6, tma=2) and L["splits"] == 1),
    ("fwd reg fp32 slabs, split > 1", lambda c, L, v: _reg(L, MODE_FWD, 6, tma=2) and L["splits"] > 1),
    ("fwd staged out_t", lambda c, L, v: _staged(L, MODE_FWD) and c.out_t),
    ("fwd staged out_f32 + bias", lambda c, L, v: _staged(L, MODE_FWD) and c.f32 == "plain" and c.bias),
    ("fwd staged N % 8 != 0", lambda c, L, v: _staged(L, MODE_FWD) and c.out and c.N % 8 != 0),
    ("fwd staged ldo % 8 != 0", lambda c, L, v: _staged(L, MODE_FWD) and c.out and c.ldo_odd),
    ("fwd staged fp32 rows not 16-byte aligned", lambda c, L, v: _staged(L, MODE_FWD) and c.f32 and c.f32_shift),
    ("fwd staged split-K slabs", lambda c, L, v: _staged(L, MODE_FWD) and c.f32 in ("slabs", "dense") and L["splits"] > 1),
    ("relu dgrad reg BN128 gate_mask / sumsq", lambda c, L, v: _reg(L, MODE_DGRAD) and (c.gate == "bits" or c.sumsq)),
    ("relu dgrad reg BN256 gate_mask / sumsq", lambda c, L, v: _reg(L, MODE_DGRAD, 4, WIDE) and (c.gate == "bits" or c.sumsq)),
    ("relu dgrad staged gate_fast", lambda c, L, v: _staged(L, MODE_DGRAD) and c.gate == "relu" and not c.ldg_odd and c.N >= 64),
    ("relu dgrad staged scalar gate, ldg % 8 != 0", lambda c, L, v: _staged(L, MODE_DGRAD) and c.gate == "relu" and c.ldg_odd),
    ("relu dgrad staged scalar gate, partial column group", lambda c, L, v: _staged(L, MODE_DGRAD) and c.gate == "relu" and c.N % 64 != 0),
    ("relu dgrad + colsum", lambda c, L, v: L["mode"] == MODE_DGRAD and c.colsum),
    ("silu dgrad gate_vec", lambda c, L, v: _staged(L, MODE_DGRAD_VEC) and not c.ldg_odd),
    ("silu dgrad scalar gate", lambda c, L, v: _staged(L, MODE_DGRAD_VEC) and c.ldg_odd),
    ("silu dgrad alpha != 1 + sumsq", lambda c, L, v: _staged(L, MODE_DGRAD_VEC) and c.alpha != 1.0 and c.sumsq),
    ("wgrad TMA reduce-add, split 1", lambda c, L, v: L["mode"] == MODE_WGRAD and L["tma_out"] == 1 and L["splits"] == 1),
    ("wgrad TMA reduce-add, split > 1", lambda c, L, v: L["mode"] == MODE_WGRAD and L["tma_out"] == 1 and L["splits"] > 1),
    ("wgrad red_stage atomics, split 1", lambda c, L, v: L["mode"] == MODE_WGRAD and L["tma_out"] == 0 and L["splits"] == 1),
    ("wgrad red_stage atomics, split > 1", lambda c, L, v: L["mode"] == MODE_WGRAD and L["tma_out"] == 0 and L["splits"] > 1),
    ("wgrad through dense.gemm: slabs + ordered sum", lambda c, L, v: c.f32 == "dense" and L["splits"] > 1),
    ("generic bias + colsum", lambda c, L, v: L["mode"] == MODE_GENERIC and c.bias and c.colsum),
    ("generic forward + accumulate", lambda c, L, v: L["mode"] == MODE_GENERIC and c.f32 == "accum" and (c.bias or c.act != "none")),
    ("generic accumulate with alpha != 1, split > 1", lambda c, L, v: L["mode"] == MODE_GENERIC and c.f32 == "accum" and c.alpha != 1.0
     and L["splits"] > 1),
] + [(f"{lay} x {MODE_NAMES[m]}", (lambda lay, m: lambda c, L, v: c.layout == lay and L["mode"] == m)(lay, m))
     for lay in ("ak_bk", "ak_bmn", "amn_bk", "amn_bmn") for m in MODE_NAMES]


def cells_of(c: Case, L: Dict[str, int], variant: str) -> List[str]:
    return [cid for cid, pred in CELLS if pred(c, L, variant)]


# The epilogues a boundary-shape case may take, one per mode (and the mode's usual companions).
_EPILOGUES = {
    "fwd": [dict(bias=True, act="relu", relu_mask=True), dict(act="silu", preact=True), dict(bias=True, alpha=0.5),
            dict(out=False, f32="plain"), dict(out=False, f32="slabs", split_k=3), dict(bias=True, out_t=True, f32="plain")],
    "dgrad": [dict(gate="bits", sumsq=True), dict(gate="relu", colsum=True), dict(alpha=0.25, sumsq=True), dict(gate="relu", ldg_odd=True)],
    "dgrad_vec": [dict(gate="silu"), dict(gate="silu", alpha=0.5, sumsq=True), dict(gate="silu", ldg_odd=True, colsum=True)],
    "wgrad": [dict(out=False, f32="accum"), dict(out=False, f32="accum", split_k=3), dict(out=False, f32="accum", ldf_odd=True, split_k=2)],
    "generic": [dict(bias=True, colsum=True), dict(bias=True, act="relu", f32="accum"), dict(out=False, f32="accum", alpha=0.5, split_k=2)],
}
BOUNDARY_M = [1, 64, 65, 127, 128, 129, 255, 257, 1000]
BOUNDARY_N = [8, 69, 120, 128, 136, 255, 256, 257, 264, 1960]
BOUNDARY_K = [8, 16, 63, 64, 65, 69, 72, 136, 960, 4160]


def boundary_cases() -> List[Case]:
    """Every boundary value of M, N and K at least once with every layout and mode (a covering set, not the cross product)."""
    out = []
    for li, (a_mn, b_mn) in enumerate([(False, False), (False, True), (True, False), (True, True)]):
        for mi, (mname, eps) in enumerate(_EPILOGUES.items()):
            for i in range(10):
                M, N, K = BOUNDARY_M[(i + li) % 9], BOUNDARY_N[i], BOUNDARY_K[(3 * i + mi + li) % 10]
                ep = eps[(i + li) % len(eps)]
                c = Case(f"edge_{'ab'[a_mn]}{'ab'[b_mn]}_{mname}_{M}x{N}x{K}", M, N, K, a_mn=a_mn, b_mn=b_mn, **ep)
                if c.sumsq:
                    K = min(K, 1024)
                    c = replace(c, K=K, name=f"edge_{'ab'[a_mn]}{'ab'[b_mn]}_{mname}_{M}x{N}x{K}")
                out.append(c)
    return out


def persistent_cases() -> List[Case]:
    """More than 132 tiles, kb_per_item 1..7 against ring depths 6 (forward), 5 (forward with pre-activation) and 4 (staged), so the
    ring's parity wraps at different points inside an item of a CTA that loops over several."""
    out = []
    for kb in range(1, 8):
        K = 64 * kb - (kb % 3) * 3          # ragged last k-block on two of three
        for depth, ep in ((6, dict(bias=True, act="relu", relu_mask=True)), (5, dict(act="silu", preact=True)),
                          (4, dict(gate="relu", colsum=True))):
            out.append(Case(f"persist_kb{kb}_s{depth}", 2048, 1280, K, b_mn=depth == 4, **ep))
    return out


def table_cases() -> List[Case]:
    """One or more hand-written cases per row of CELLS (on an H100's 132 SMs)."""
    C = Case
    return [
        C("fwd_bias_s6", 300, 264, 136, bias=True, alpha=0.5, cell="fwd reg bf16 S6 BN128 + bias"),
        C("fwd_relu_mask_s6", 257, 136, 960, act="relu", relu_mask=True, bias=True, cell="fwd reg bf16 S6 BN128 + relu + mask words"),
        C("fwd_silu_s6", 129, 256, 72, act="silu", bias=True, cell="fwd reg bf16 S6 BN128 + silu"),
        C("fwd_preact_s5", 255, 264, 65, act="silu", preact=True, bias=True, cell="fwd reg bf16 + preact S5"),
        C("fwd_wide_bk", 2048, 1280, 256, bias=True, act="relu", relu_mask=True, cell="fwd reg bf16 BN256, B K-major"),
        C("fwd_wide_bmn", 2000, 1960, 320, b_mn=True, act="relu", cell="fwd reg bf16 BN256, B MN-major"),
        C("fwd_f32_split1", 1000, 264, 960, out=False, f32="plain", cell="fwd reg fp32 slabs, split 1"),
        C("fwd_f32_slabs", 257, 120, 4160, out=False, f32="slabs", split_k=6, cell="fwd reg fp32 slabs, split > 1"),
        C("fwd_f32_slabs_amn", 129, 256, 1000, a_mn=True, b_mn=True, out=False, f32="slabs", split_k=4, cell="fwd reg fp32 slabs, split > 1"),
        C("fwd_staged_out_t", 257, 255, 136, bias=True, act="relu", out_t=True, cell="fwd staged out_t"),
        C("fwd_staged_f32_bias", 300, 264, 200, bias=True, alpha=0.25, f32="plain", cell="fwd staged out_f32 + bias"),
        C("fwd_staged_n69", 1000, 69, 960, bias=True, act="relu", relu_mask=True, cell="fwd staged N % 8 != 0"),
        C("fwd_staged_ldo_odd", 129, 264, 72, act="silu", preact=True, ldo_odd=True, cell="fwd staged ldo % 8 != 0"),
        C("fwd_staged_f32_unaligned", 65, 136, 69, out=False, f32="plain", f32_shift=True, cell="fwd staged fp32 rows not 16-byte aligned"),
        C("fwd_staged_slabs_odd", 127, 257, 1000, out=False, f32="slabs", split_k=3, cell="fwd staged split-K slabs"),
        C("dgrad_bits_s6", 1000, 264, 512, b_mn=True, gate="bits", sumsq=True, cell="relu dgrad reg BN128 gate_mask / sumsq"),
        C("dgrad_bits_wide", 2048, 1280, 320, b_mn=True, gate="bits", cell="relu dgrad reg BN256 gate_mask / sumsq"),
        C("dgrad_sumsq_wide", 2048, 1280, 256, alpha=0.25, sumsq=True, cell="relu dgrad reg BN256 gate_mask / sumsq"),
        C("dgrad_gate_fast", 300, 1000, 72, b_mn=True, gate="relu", cell="relu dgrad staged gate_fast"),
        C("dgrad_gate_scalar", 257, 264, 136, b_mn=True, gate="relu", ldg_odd=True, cell="relu dgrad staged scalar gate, ldg % 8 != 0"),
        C("dgrad_gate_partial", 300, 200, 136, gate="relu", sumsq=True, cell="relu dgrad staged scalar gate, partial column group"),
        C("dgrad_colsum", 1000, 264, 69, b_mn=True, gate="relu", colsum=True, cell="relu dgrad + colsum"),
        C("dgrad_vec", 300, 264, 136, b_mn=True, gate="silu", cell="silu dgrad gate_vec"),
        C("dgrad_vec_scalar", 129, 136, 72, gate="silu", ldg_odd=True, cell="silu dgrad scalar gate"),
        C("dgrad_vec_gp", 1000, 1960, 512, b_mn=True, gate="silu", alpha=0.25, sumsq=True, cell="silu dgrad alpha != 1 + sumsq"),
        C("wgrad_tma", 264, 136, 1000, a_mn=True, b_mn=True, out=False, f32="accum", cell="wgrad TMA reduce-add, split 1"),
        C("wgrad_tma_split", 256, 264, 4160, a_mn=True, b_mn=True, out=False, f32="accum", split_k=5, cell="wgrad TMA reduce-add, split > 1"),
        C("wgrad_atomic", 136, 69, 1000, a_mn=True, b_mn=True, out=False, f32="accum", ldf_odd=True, cell="wgrad red_stage atomics, split 1"),
        C("wgrad_atomic_split", 120, 257, 4160, a_mn=True, b_mn=True, out=False, f32="accum", f32_shift=True, split_k=4,
          cell="wgrad red_stage atomics, split > 1"),
        C("wgrad_dense", 264, 255, 4160, a_mn=True, b_mn=True, out=False, f32="dense", split_k=4, cell="wgrad through dense.gemm: slabs + ordered sum"),
        C("wgrad_dense_n4", 69, 136, 1000, a_mn=True, b_mn=True, out=False, f32="dense", split_k=3, cell="wgrad through dense.gemm: slabs + ordered sum"),
        C("generic_bias_colsum", 257, 264, 136, bias=True, colsum=True, cell="generic bias + colsum"),
        C("generic_fwd_accum", 300, 136, 960, bias=True, act="relu", f32="accum", cell="generic forward + accumulate"),
        C("generic_accum_alpha", 128, 256, 4160, a_mn=True, b_mn=True, out=False, f32="accum", alpha=0.5, split_k=3,
          cell="generic accumulate with alpha != 1, split > 1"),
    ]


def random_cases(n: int = 100, seed: int = 20261019) -> List[Case]:
    """A seeded draw of shapes, layouts and epilogues from the same legal space."""
    r = random.Random(seed)
    eps = [e for v in _EPILOGUES.values() for e in v]
    out = []
    for i in range(n):
        ep = dict(r.choice(eps))
        M, N = r.choice(BOUNDARY_M + [r.randint(1, 1200)]), r.choice(BOUNDARY_N + [r.randint(1, 1200)])
        K = r.choice(BOUNDARY_K + [r.randint(1, 2100)])
        if ep.get("sumsq"):
            K = min(K, 1024)
        for knob in ("ldo_odd", "ldf_odd", "f32_shift", "ldg_odd"):
            if r.random() < 0.15:
                ep[knob] = True
        if ep.get("f32") in ("slabs", "accum") and ep.get("out") is False and r.random() < 0.5:      # split-K: plain fp32 only
            ep["split_k"] = r.randint(1, 6)
        out.append(Case(f"rand{i:03d}_{M}x{N}x{K}", M, N, K, a_mn=r.random() < 0.5, b_mn=r.random() < 0.5, **ep))
    return out


def all_cases() -> List[Case]:
    return table_cases() + persistent_cases() + boundary_cases() + random_cases()


# ---------------------------------------------------------------------------------------------------------------------- buffers
def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64, torch.int32: torch.int32}[t.dtype])


class Guarded:
    """A strided window (shape, strides, element offset `base`) of a flat buffer of `total` elements that holds `sentinel` bits
    everywhere else.  check() raises when anything outside the window changed."""

    def __init__(self, name, shape, strides, base, total, dtype, sentinel, device, fill=None):
        self.name = name
        self.flat = torch.empty(total, dtype=dtype, device=device)
        _bits(self.flat).fill_(sentinel)
        self.view = self.flat.as_strided(shape, strides, base)
        if fill is not None:
            self.view.copy_(fill)
        self.inside = torch.zeros(total, dtype=torch.bool, device=device)
        self.inside.as_strided(shape, strides, base).fill_(True)
        self.before = self.flat.clone()

    def check(self, rep: Optional[Report], link: str) -> None:
        bad = (_bits(self.flat) != _bits(self.before)) & ~self.inside
        if rep is not None:
            rep.add(link + " guard band", float(bad.any()))
        if bad.any():
            k = int(torch.nonzero(bad)[0])
            raise BoundError(f"{link} guard band: {int(bad.sum())} elements outside the window changed; first at flat index {k} (window base "
                             f"{self.view.storage_offset()}, strides {self.view.stride()})")


def _c8(x):
    return _ceil(x, 8) * 8


def _c4(x):
    return _ceil(x, 4) * 4


def bf16_window(name, rows, cols, odd, device):
    ld = _c8(8 + cols) + 8 + (3 if odd else 0)
    return Guarded(name, (rows, cols), (ld, 1), 2 * ld + 8, (rows + 5) * ld, torch.bfloat16, BF16_SENTINEL, device)


def f32_window(name, rows, cols, odd, shift, device, fill=None):
    ld = _c4(4 + cols) + 4 + (1 if odd else 0)
    return Guarded(name, (rows, cols), (ld, 1), 2 * ld + 4 + int(shift), (rows + 5) * ld, torch.float32, 0x7FC00000, device, fill)


def slab_window(name, splits, rows, cols, odd, shift, device):
    """splits + 1 slabs allocated: the one past pulse_gemm_num_splits must keep its sentinel."""
    ld = _c4(4 + cols) + 4 + (1 if odd else 0)
    stride = (rows + 2) * ld
    return Guarded(name, (splits, rows, cols), (stride, ld, 1), ld + 4 + int(shift), (splits + 1) * stride + 2 * ld, torch.float32,
                   0x7FC00000, device)


def operand(vals: torch.Tensor, mn: bool) -> torch.Tensor:
    """bf16 operand for logical [rows, K] values: K-major [rows, lda] or MN-major [K, lda]; padding columns and four extra rows of NaN."""
    src = vals.T if mn else vals
    r, c = src.shape
    buf = torch.empty(r + 4, _c8(c) + 8, dtype=torch.bfloat16, device=vals.device)
    _bits(buf).fill_(BF16_NAN)
    buf[:r, :c] = src.to(torch.bfloat16)
    return buf[:r, :c]


def _pattern(rows, cols, p, a, b, c, off, device):
    i = torch.arange(rows, device=device, dtype=torch.int64)[:, None]
    j = torch.arange(cols, device=device, dtype=torch.int64)[None, :]
    return ((a * i + b * j + c * i * j + off * 1) % p - p // 2).to(torch.float64)


def sumsq_exact(v: torch.Tensor, alpha: float) -> bool:
    """Every fp32 partial sum of squares the kernel forms (one warp: at most 32 rows x 128 columns, aligned) is exact: the squares of
    the values in units of alpha^2 add up to less than 2^24 in every aligned 32 x 128 block."""
    M, N = v.shape
    q = torch.zeros(_ceil(M, 32) * 32, _ceil(N, 128) * 128, dtype=torch.float64, device=v.device)
    q[:M, :N] = (v / alpha) ** 2
    blocks = q.view(q.shape[0] // 32, 32, q.shape[1] // 128, 128).sum((1, 3))
    return bool((blocks < 2.0 ** 24).all())


class Operands:
    """The inputs of one case in one family: logical fp64 values (A [M, K], B [K, N], bias, gate) and the device buffers."""

    def __init__(self, c: Case, exact: bool, device, seed: int = 0):
        M, N, K = c.M, c.N, c.K
        self.exact = exact
        g = torch.Generator(device="cpu").manual_seed(seed + 7919 * M + 104729 * N + 31 * K)
        if exact:
            a = _pattern(M, K, 17, 31, 7, 3, seed, device)                                  # [-8, 8]
            b = _pattern(K, N, 17, 11, 13, 5, seed + 5, device)
            if c.sumsq and not sumsq_exact(a.to(torch.bfloat16).double() @ b.to(torch.bfloat16).double(), 1.0):
                # [-2, 2], B with at most 12 non-zeros per column: |acc| <= 48, so 4096 squares stay below 2^24
                p = max(8, _ceil(K, 12))
                a = _pattern(M, K, 5, 3, 1, 1, seed, device)
                b = _pattern(K, N, 5, 1, 2, 1, seed + 1, device) * ((torch.arange(K, device=device)[:, None] + 3 *
                                                                    torch.arange(N, device=device)[None, :]) % p == 0)
            bias = _pattern(1, N, 23, 1, 7, 0, seed, device)[0]
            gate = {"relu": _pattern(M, N, 7, 5, 3, 1, seed, device), "silu": _pattern(M, N, 17, 3, 5, 1, seed, device) / 4}.get(c.gate)
        else:
            a = torch.randn(M, K, generator=g, dtype=torch.float64).to(device)
            b = (torch.randn(K, N, generator=g, dtype=torch.float64) / math.sqrt(K)).to(device)
            bias = torch.randn(N, generator=g, dtype=torch.float64).to(device)
            gate = torch.randn(M, N, generator=g, dtype=torch.float64).to(device) if c.gate in ("relu", "silu") else None
        if gate is not None and c.gate == "relu":                                          # exact zeros, -0.0 and tiny positives
            gate[::3] = torch.relu(gate[::3])
            gate[1::7, ::5] = -0.0
            gate[2::11, 1::4] = 1e-30
        self.a = a.to(torch.bfloat16).to(torch.float64)
        self.b = b.to(torch.bfloat16).to(torch.float64)
        self.A = operand(self.a, c.a_mn)                   # [M, K] K-major or [K, M] MN-major
        self.B = operand(self.b.T, c.b_mn)                 # [N, K] K-major or [K, N] MN-major
        self.bias = self.bias_buf = None
        if c.bias:
            self.bias_buf = torch.full((N + 8,), float("nan"), device=device)
            self.bias_buf[:N] = bias.float()
            self.bias = self.bias_buf[:N]
        self.gate = self.gate_buf = None
        if gate is not None:
            ldg = _c8(N) + 8 + (1 if c.ldg_odd else 0)
            buf = torch.empty(M + 4, ldg, dtype=torch.bfloat16, device=device)
            _bits(buf).fill_(BF16_NAN)
            buf[:M, :N] = gate.to(torch.bfloat16)
            self.gate = buf[:M, :N]
        self.gate_words = None
        if c.gate == "bits":
            W = _ceil(N, 32)
            words = torch.randint(-2 ** 31, 2 ** 31 - 1, (W + 1, M + 5), generator=g, dtype=torch.int32).to(device)
            self.gate_words = words[:W, :M]

    def gate_bits(self, N: int) -> torch.Tensor:
        return unpack_mask(self.gate_words, N, self.gate_words.shape[1])


class Outputs:
    """The guarded output buffers of a case."""

    def __init__(self, c: Case, ops: Operands, device):
        M, N = c.M, c.N
        self.out = bf16_window("out", M, N, c.ldo_odd, device) if c.out else None
        self.preact = bf16_window("preact", M, N, c.ldo_odd, device) if c.preact else None
        self.out_t = bf16_window("out_t", N, M, c.ldo_odd, device) if c.out_t else None
        self.f32 = self.f32_init = None
        ns = num_splits(c.K, c.split_k)
        if c.f32 == "slabs":
            self.f32 = slab_window("slabs", ns, M, N, c.ldf_odd, c.f32_shift, device)
        elif c.f32:
            init = None
            if c.f32 in ("accum", "dense"):               # accumulate adds to what is there: integer start values
                init = _pattern(M, N, 9, 1, 1, 0, 0, device).float()
                self.f32_init = init.double()
            self.f32 = f32_window("out_f32", M, N, c.ldf_odd, c.f32_shift, device, fill=init)
        self.colsum = self.colsum_init = None
        if c.colsum:
            self.colsum_init = _pattern(1, N, 5, 0, 1, 0, 0, device)[0]
            self.colsum = Guarded("colsum", (N,), (1,), 2, N + 10, torch.float32, 0x7FC00000, device, fill=self.colsum_init.float())
        self.sumsq = None
        if c.sumsq:
            self.sumsq = Guarded("sumsq", (1,), (1,), 1, 3, torch.float64, 0x7FF8000000000000, device,
                                 fill=torch.ones(1, dtype=torch.float64))
        self.mask = None
        if c.relu_mask:
            W = _ceil(N, 32)
            self.mask = Guarded("relu_mask", (W, M), (M + 5, 1), M + 5 + 3, (W + 2) * (M + 5), torch.int32, MASK_SENTINEL, device)


# ------------------------------------------------------------------------------------------------------------------- reference
class Expected:
    """fp64 reference of a case's final values (v: after alpha, bias, activation and gate, before any output rounding) with its
    bound; tol == 0 where the family makes the value exact."""

    def __init__(self, c: Case, ops: Operands):
        a, b = ops.a, ops.b
        bias = f64(ops.bias) if ops.bias is not None else None
        acc = a @ b
        self.pre = c.alpha * acc + (bias if bias is not None else 0.0)
        self.pre_exact = ops.exact
        self.g_pre = None if ops.exact else Gemm(c.alpha * a, b, bias=bias)
        v, exact = self.pre, ops.exact
        tol = torch.zeros_like(v) if exact else self.g_pre.tol(False)
        self.silu = False
        if c.act == "relu":
            v = torch.relu(v)
        elif c.act == "silu":
            g = self.g_pre or Gemm(c.alpha * a, b, bias=bias)
            v, tol, exact, self.silu = silu64(v), silu_gemm_tol(g), False, True
        if c.gate == "relu":
            keep = (f64(ops.gate) > 0).to(torch.float64)
            v, tol = v * keep, tol * keep
        elif c.gate == "bits":
            keep = ops.gate_bits(c.N).to(torch.float64)
            v, tol = v * keep, tol * keep
        elif c.gate == "silu":
            g = self.g_pre or Gemm(c.alpha * a, b, bias=bias)
            v, acc_t = silu_gated(g, ops.gate)
            tol, exact = acc_t, False
        self.v, self.tol32, self.exact = v, tol, exact
        # bf16 outputs: one more rounding (the SiLU bound has its own)
        self.tol16 = tol if self.silu else tol * (1 + UBF) + UBF * v.abs()
        if exact:
            assert bool((v.float().double() == v).all()), "exact family: a final value is not representable in fp32"


def _check_bf16(rep, link, got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, exact: bool) -> None:
    if exact:
        want = ref.float().to(torch.bfloat16)
        gb, wb = _bits(got.contiguous()).clone(), _bits(want).clone()
        gb[gb == -32768] = 0                                # -0.0 and +0.0 are the same value
        wb[wb == -32768] = 0
        bad = gb != wb
        if rep is not None:
            rep.add(link + " (bf16 RNE bits)", float(bad.any()))
        if bad.any():
            r, cc = (int(i) for i in torch.nonzero(bad)[0])
            raise BoundError(f"{link}: {int(bad.sum())} bf16 outputs differ from round-to-nearest-even; first at ({r}, {cc}): got "
                             f"{float(got[r, cc])!r} (bits {int(gb[r, cc]) & 0xFFFF:#06x}), exact {float(ref[r, cc])!r} -> "
                             f"{float(want[r, cc])!r} (bits {int(wb[r, cc]) & 0xFFFF:#06x})")
    else:
        check(rep, link, got, ref, tol)


def _check_f32(rep, link, got, ref, tol, exact) -> None:
    if exact:
        check_exact(rep, link, got, ref)
    else:
        check(rep, link, got, ref, tol)


def check_outputs(rep: Optional[Report], c: Case, ops: Operands, outs: Outputs, ref: Expected, slabs_sum=None) -> None:
    """Every output of the case against the reference, then every guard band.  Raises BoundError naming the link."""
    M, N, K = c.M, c.N, c.K
    ex = ref.exact
    if outs.out is not None:
        _check_bf16(rep, "out (bf16)", outs.out.view, ref.v, ref.tol16, ex)
    if outs.out_t is not None:
        _check_bf16(rep, "out_t (bf16, transposed)", outs.out_t.view.T, ref.v, ref.tol16, ex)
    if outs.preact is not None:
        if ref.pre_exact:
            _check_bf16(rep, "preact (bf16)", outs.preact.view, ref.pre, None, True)
        else:
            ref.g_pre.check(rep, "preact (bf16)", outs.preact.view)
    if outs.mask is not None:
        words = outs.mask.view
        if ref.pre_exact:
            W = words.shape[0]
            bits = unpack_mask(words, W * 32, M)
            if bits[:, N:].any():
                raise BoundError(f"relu_mask: mask bits set past column {N}")
            bad = bits[:, :N] != (ref.pre > 0)
            if rep is not None:
                rep.add("relu_mask (exact, y == 0 included)", float(bad.any()))
            if bad.any():
                r, cc = (int(i) for i in torch.nonzero(bad)[0])
                raise BoundError(f"relu_mask: {int(bad.sum())} bits differ from y > 0; first at row {r} column {cc} (y {float(ref.pre[r, cc])!r})")
        else:
            check_mask(rep, "relu_mask", words, ref.g_pre, N, M)
    if c.f32 == "slabs":
        ns = num_splits(K, c.split_k)
        for z in range(ns):
            k0, k1 = slab_range(K, c.split_k, z)
            part = c.alpha * (ops.a[:, k0:k1] @ ops.b[k0:k1])
            link = f"slab {z} of {ns} (k {k0}..{k1})"
            if ops.exact:
                check_exact(rep, link, outs.f32.view[z], part)
            else:
                Gemm(c.alpha * ops.a[:, k0:k1], ops.b[k0:k1]).check(rep, link, outs.f32.view[z])
    elif c.f32 in ("accum", "dense"):
        want = outs.f32_init + ref.v
        tol = ref.tol32 + U32 * want.abs() if not ex else None
        _check_f32(rep, "out_f32 (accumulated)", outs.f32.view, want, tol, ex)
    elif c.f32:
        _check_f32(rep, "out_f32", outs.f32.view, ref.v, ref.tol32, ex)
    vf = ref.v
    if outs.colsum is not None:
        want = outs.colsum_init + vf.sum(0)
        tol = None if ex else ref.tol32.sum(0) + sum_tol(vf.abs().sum(0) + outs.colsum_init.abs(), M + 1) + U32 * want.abs()
        _check_f32(rep, "colsum", outs.colsum.view, want, tol, ex)
    if outs.sumsq is not None:
        want = 1.0 + (vf * vf).sum()
        if ex:
            assert sumsq_exact(vf, c.alpha), "exact family: the case's sum of squares is not exact in fp32 partials"
            check_exact(rep, "sumsq", outs.sumsq.view[0], want)
        else:
            t = ref.tol32
            tol = (2 * vf.abs() * t + t * t).sum() + sum_tol((vf * vf).sum(), 4096) + U32 * want
            check(rep, "sumsq", outs.sumsq.view[0], want, tol)
    if slabs_sum is not None:
        got, host = slabs_sum
        check_exact(rep, "ordered_sum_add (slab order)", got, host)
    for name in ("out", "out_t", "preact", "f32", "colsum", "sumsq", "mask"):
        gbuf = getattr(outs, name)
        if gbuf is not None:
            gbuf.check(rep, gbuf.name)


def ordered_sum_host(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """pulse_ordered_sum_add (mlp_ops.cu ordered_sum_kernel) on the host: s = 0; s += x[k] for k = 0..n-1 in fp32; out + s."""
    s = torch.zeros_like(out, dtype=torch.float32)
    for k in range(x.shape[0]):
        s = s + x[k].float()
    return out.float() + s


def column_sum_host(y: torch.Tensor, out: torch.Tensor, chunk: int = 64) -> torch.Tensor:
    """dense.column_sum_add on the host: rows in chunks of `chunk` summed in row order, then the chunk sums in chunk order."""
    rows = y.shape[0]
    parts = torch.stack([ordered_sum_host(y[r:r + chunk].float(), torch.zeros(y.shape[1], device=y.device)) for r in range(0, rows, chunk)])
    return ordered_sum_host(parts, out)
