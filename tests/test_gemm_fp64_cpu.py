"""The GEMM cell checks of tests/gemm_fp64.py have teeth (no GPU needed).

A CPU simulation of the kernel -- fp32 accumulation of the bf16 operands over 64-wide k-blocks (fp64_ref.kernel_gemm), then the
epilogue's fp32 operations in the kernel's order (alpha, bias, pre-activation and mask words, activation, gate, outputs) -- writes each
case's guarded buffers as the kernel would.  It must pass every hand-written cell case in both operand families, and each mutation
below, a bug the GPU suite is there to catch, must be rejected with the link it breaks.
"""
import pytest
import torch

from tests import gemm_fp64 as gf
from tests.fp64_ref import BoundError, kernel_gemm, pack_mask

DEV = "cpu"


def _pad_col(t: torch.Tensor, k: int, mn: bool) -> torch.Tensor:
    """Reduction index k of an operand read from its allocation (past the logical extent: the NaN padding)."""
    buf = t._base
    return buf[k, :t.shape[1]].double() if mn else buf[:t.shape[0], k].double()


def simulate(c: gf.Case, ops: gf.Operands, outs: gf.Outputs, mut: str = ""):
    """Writes the outputs of case c into outs as the kernel does; `mut` injects one bug.  Returns the ordered-sum pair for slab cases
    (the device sum and the host model of it: here both come from the host)."""
    M, N, K = c.M, c.N, c.K
    a, b = ops.a, ops.b
    kuse = K // 64 * 64 if mut == "drop_last_partial_kblock" else K
    acc = kernel_gemm(a[:, :kuse], b[:kuse])
    if mut == "skip_k16":
        acc[:128, :128] -= (a[:128, 16:32].float() @ b[16:32, :128].float())
    if mut == "pad_column_read":
        acc = acc + (_pad_col(ops.A, K, c.a_mn)[:, None] * _pad_col(ops.B, K, c.b_mn)[None, :]).float()
    alpha = torch.tensor(c.alpha, dtype=torch.float32)
    bias = ops.bias.float() if ops.bias is not None else None
    if mut == "alpha_bias" and bias is not None:
        v = (acc + bias) * alpha
    else:
        v = acc * alpha
        if bias is not None:
            v = v + bias
    pre = v
    if c.act == "relu":
        v = torch.relu(v)
    elif c.act == "silu":
        v = v / (1 + torch.exp(-v))
    if c.gate == "relu":
        g = ops.gate.float()
        if mut == "gate_stride_n":
            g = ops.gate._base.reshape(-1)[:M * N].reshape(M, N).float()
        v = v * (g > 0)
    elif c.gate == "bits":
        v = v * ops.gate_bits(N)
    elif c.gate == "silu":
        z = ops.gate.float()
        s = 1 / (1 + torch.exp(-z))
        v = v * (s * (1 + z * (1 - s)))
    if outs.out is not None:
        y = v.to(torch.bfloat16)
        if mut == "bf16_trunc":
            y = (gf._bits(v.contiguous()) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)
        outs.out.view.copy_(y)
        if mut == "store_past_n":
            outs.out.flat[outs.out.view.storage_offset() + N] = 0
    if outs.out_t is not None:
        outs.out_t.view.copy_(v.T.to(torch.bfloat16))
        if mut == "out_t_tail":
            n0 = (N - 1) // 128 * 128
            outs.out_t.view[n0:, 1:] = v.T[n0:, :-1].to(torch.bfloat16)
    if outs.preact is not None:
        outs.preact.view.copy_(pre.to(torch.bfloat16))
    if outs.mask is not None:
        bits = pre >= 0 if mut == "mask_at_zero" else pre > 0
        words = pack_mask(bits)
        if mut == "mask_past_n":
            words[-1] |= 1 << (N % 32)
        outs.mask.view.copy_(words)
    slabs_sum = None
    if c.f32 == "slabs":
        ns = gf.num_splits(K, c.split_k)
        parts = []
        for z in range(ns):
            k0, k1 = gf.slab_range(K, c.split_k, z)
            if mut == "slab_shift" and z == 1:
                k0, k1 = k0 + 64, min(K, k1 + 64)
            parts.append(kernel_gemm(a[:, k0:k1], b[k0:k1]) * alpha)
        if mut == "slab_index":
            parts[0], parts[1] = parts[1], parts[0]
        for z, p in enumerate(parts):
            outs.f32.view[z].copy_(p)
        host = gf.ordered_sum_host(outs.f32.view[:ns], torch.zeros(M, N))
        slabs_sum = (host.clone(), host)
    elif c.f32 in ("accum", "dense"):
        if mut == "accum_overwrite":
            outs.f32.view.copy_(v)
        else:
            extra = 0
            if mut == "split_twice":
                k0, k1 = gf.slab_range(K, c.split_k, 1)
                extra = kernel_gemm(a[:, k0:k1], b[k0:k1]) * alpha
            outs.f32.view.add_(v + extra)
    elif c.f32:
        outs.f32.view.copy_(v.to(torch.bfloat16).float() if mut == "f32_via_bf16" else v)
    if outs.colsum is not None:
        cs = v.sum(0)
        if mut == "colsum_extra_row":                  # row M's value, from row M of A's allocation (the NaN padding)
            buf = ops.A._base
            row_m = buf[:K, M] if c.a_mn else buf[M, :K]
            cs = cs + (row_m.float() @ b.float()) * alpha
        outs.colsum.view.add_(cs)
    if outs.sumsq is not None:
        w = v.to(torch.bfloat16) if mut == "sumsq_bf16" else v
        outs.sumsq.view.add_((w.double() ** 2).sum())
    return slabs_sum


def _run(c: gf.Case, exact: bool, mut: str = "", rep=None):
    ops = gf.Operands(c, exact, DEV)
    outs = gf.Outputs(c, ops, DEV)
    ss = simulate(c, ops, outs, mut)
    gf.check_outputs(rep, c, ops, outs, gf.Expected(c, ops), slabs_sum=ss)


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("case", gf.table_cases(), ids=lambda c: c.name)
def test_simulated_kernel_passes_every_cell(case, exact):
    _run(case, exact)


def test_cell_cases_reach_their_cells_on_132_sms():
    """Each hand-written case lands in the CELLS row it names under the default dispatch of an H100, and the whole case list reaches
    every row (the GPU suite asserts the same against pulse_gemm_last_launch)."""
    reached = set()
    for c in gf.all_cases():
        for v in gf.VARIANTS:
            L = gf.predict(c, gf.H100_SMS, v)
            cells = gf.cells_of(c, L, v)
            reached.update(cells)
            if v == "default" and c.cell:
                assert c.cell in cells, f"{c.name} is meant for '{c.cell}' but the dispatch model puts it in {gf.cell_name(c, L)}"
    assert [cid for cid, _ in gf.CELLS if cid not in reached] == []


def test_dispatch_model_matches_known_launches():
    """predict() against launches whose kernels DESIGN.md names: the update's wide forward, the K = 69 head dgrad (narrow), the
    discriminator's M = 12288, N = 512 forward (narrow: 192 wide items are 2 rounds against 3), the split-K slabs (register fp32)."""
    C = gf.Case
    L = gf.predict(C("", 16384, 1024, 960, act="relu", relu_mask=True), 132)
    assert (L["mode"], L["stages"], L["tile_n"], L["tma_out"], L["grid"]) == (gf.MODE_FWD, 4, 256, 1, 132)
    assert gf.predict(C("", 16384, 512, 69, b_mn=True, gate="bits"), 132)["tile_n"] == 128
    assert gf.predict(C("", 12288, 512, 1024, act="relu"), 132)["tile_n"] == 128
    L = gf.predict(C("", 1024, 960, 16384, a_mn=True, b_mn=True, out=False, f32="slabs", split_k=8), 132)
    assert (L["mode"], L["stages"], L["tma_out"], L["splits"]) == (gf.MODE_FWD, 6, 2, 8)
    assert gf.predict(C("", 1024, 960, 16384, out=False, f32="slabs", split_k=8), 132, "stages4")["tma_out"] == 0
    assert gf.predict(C("", 64, 64, 64, out=False, f32="accum", alpha=0.5), 132)["mode"] == gf.MODE_GENERIC
    assert gf.num_splits(4160, 6) == 6 and gf.slab_range(4160, 6, 5) == (3520, 4160) and gf.num_splits(130, 3) == 3
    assert gf.num_splits(200, 6) == 4


# (mutation, case, family, the link that must reject it)
C = gf.Case
MUTANTS = [
    ("drop_last_partial_kblock", C("k65", 129, 136, 65, bias=True), True, "out (bf16)"),
    ("drop_last_partial_kblock", C("k69", 65, 120, 69, out=False, f32="plain"), True, "out_f32"),
    ("drop_last_partial_kblock", C("k69b", 65, 120, 69, out=False, f32="plain"), False, "out_f32"),
    ("skip_k16", C("k16", 257, 264, 136), True, "out (bf16)"),
    ("skip_k16", C("k16b", 257, 264, 136, out=False, f32="plain"), False, "out_f32"),
    ("slab_shift", C("slabs", 129, 136, 1000, out=False, f32="slabs", split_k=4), True, "slab 1"),
    ("slab_index", C("slabs", 129, 136, 1000, out=False, f32="slabs", split_k=4), True, "slab 0"),
    ("split_twice", C("acc", 64, 136, 1000, a_mn=True, b_mn=True, out=False, f32="accum", split_k=3), True, "out_f32 (accumulated)"),
    ("bf16_trunc", C("rne", 257, 264, 960), True, "out (bf16)"),
    ("f32_via_bf16", C("f32", 257, 264, 960, out=False, f32="plain"), True, "out_f32"),
    ("f32_via_bf16", C("f32b", 257, 264, 960, out=False, f32="plain"), False, "out_f32"),
    ("mask_at_zero", C("mask0", 257, 264, 136, bias=True, act="relu", relu_mask=True), True, "relu_mask"),
    ("mask_past_n", C("mask69", 65, 69, 136, act="relu", relu_mask=True), True, "relu_mask"),
    ("mask_past_n", C("mask69b", 65, 69, 136, act="relu", relu_mask=True), False, "relu_mask"),
    ("colsum_extra_row", C("cs", 129, 136, 136, gate="relu", colsum=True), True, "colsum"),
    ("sumsq_bf16", C("ss", 33, 8, 32, alpha=0.25, sumsq=True), True, "sumsq"),
    ("accum_overwrite", C("ow", 64, 136, 1000, a_mn=True, b_mn=True, out=False, f32="accum"), True, "out_f32 (accumulated)"),
    ("gate_stride_n", C("gs", 129, 136, 136, b_mn=True, gate="relu"), True, "out (bf16)"),
    ("alpha_bias", C("ab", 129, 136, 136, bias=True, alpha=0.5), True, "out (bf16)"),
    ("alpha_bias", C("abb", 129, 136, 136, bias=True, alpha=0.5), False, "out (bf16)"),
    ("out_t_tail", C("ot", 129, 200, 136, out_t=True, bias=True), True, "out_t"),
    ("store_past_n", C("pastn", 65, 136, 72), True, "out guard band"),
    ("pad_column_read", C("pad", 65, 136, 72), True, "out (bf16)"),
    ("pad_column_read", C("padmn", 65, 136, 72, a_mn=True, b_mn=True), False, "out (bf16)"),
]


@pytest.mark.parametrize("mut,case,exact,link", MUTANTS, ids=[f"{m[0]}-{m[1].name}-{'exact' if m[2] else 'bounded'}" for m in MUTANTS])
def test_mutant_is_rejected(mut, case, exact, link):
    _run(case, exact)                          # the case itself passes
    with pytest.raises(BoundError) as e:
        _run(case, exact, mut)
    assert str(e.value).startswith(link) or link in str(e.value).split(":")[0], str(e.value)


def test_guard_band_and_slab_sentinels_are_checked():
    """A slab past pulse_gemm_num_splits that was written, and a mask word row past M, are guard-band violations."""
    c = C("slabs", 129, 136, 1000, out=False, f32="slabs", split_k=4)
    ops = gf.Operands(c, True, DEV)
    outs = gf.Outputs(c, ops, DEV)
    simulate(c, ops, outs)
    ns = gf.num_splits(c.K, c.split_k)
    outs.f32.view.as_strided((c.M, c.N), outs.f32.view.stride()[1:], outs.f32.view.storage_offset() + ns * outs.f32.view.stride(0)).fill_(0)
    with pytest.raises(BoundError, match="slabs guard band"):
        gf.check_outputs(None, c, ops, outs, gf.Expected(c, ops))
    c = C("mask", 65, 69, 136, act="relu", relu_mask=True)
    ops = gf.Operands(c, True, DEV)
    outs = gf.Outputs(c, ops, DEV)
    simulate(c, ops, outs)
    outs.mask.flat[outs.mask.view.storage_offset() + c.M] = 0
    with pytest.raises(BoundError, match="relu_mask guard band"):
        gf.check_outputs(None, c, ops, outs, gf.Expected(c, ops))


def test_ordered_sums_host_order():
    """ordered_sum_host adds the slabs in slice order (0 + x0 + x1 + ...), column_sum_host rows in 64-row chunks then the chunks: both
    differ from a reordered fp32 sum on data where the order matters."""
    x = torch.tensor([[[1.0]], [[2.0 ** 24]], [[1.0]], [[-2.0 ** 24]]])
    assert float(gf.ordered_sum_host(x, torch.zeros(1, 1))) == 0.0          # 1 + 2^24 rounds to 2^24
    assert float(gf.ordered_sum_host(x.flip(0), torch.zeros(1, 1))) == 2.0
    y = torch.ones(130, 1)
    y[64] = 2.0 ** 24
    assert float(gf.column_sum_host(y, torch.zeros(1))) == 2.0 ** 24 + 66      # chunks 64, 2^24 (63 ones lost), 2
    assert float(gf.ordered_sum_host(y[:, None], torch.zeros(1, 1))) == 2.0 ** 24 + 64     # one pass in row order loses 65
