"""The deep-ring GEMM kernels (6 stages, 5 with a pre-activation; register-resident epilogue only) against the 4-stage kernel
(PULSE_GEMM_STAGES=4): the tile, the warp roles and the MMA order are the same, so every output must match bit for bit; only the
fp64 sum of squares, added by atomics in scheduling order, may differ in its last bits."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _bf(g, r, c, scale=1.0):
    """bf16 [r, c] view with rows padded to 16 bytes (the GEMM's operand alignment)"""
    return (torch.randn(r, (c + 7) // 8 * 8, device=DEV, generator=g) * scale).bfloat16()[:, :c]


def _both(monkeypatch, run):
    """run() with the 4-stage kernel, then with the default (deep-ring) one; returns both results"""
    monkeypatch.setenv("PULSE_GEMM_STAGES", "4")
    ref = run()
    monkeypatch.delenv("PULSE_GEMM_STAGES")
    new = run()
    torch.cuda.synchronize()
    return ref, new


def _same(x: torch.Tensor, y: torch.Tensor) -> bool:
    return torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x, y.view(torch.int16) if y.dtype == torch.bfloat16 else y)


# (M, N, K): the update's forward shapes, row tails (4096 / 1000) and a column tail (N = 200)
FWD = [(16384, 1024, 960), (16384, 512, 1024), (12288, 1024, 1984), (4096, 1024, 1960), (1000, 512, 960), (1000, 200, 136)]


@pytest.mark.parametrize("M,N,K", FWD)
def test_forward_relu_mask_words(monkeypatch, M, N, K):
    from pulse_b200.dense import gemm_nt
    g = torch.Generator(device=DEV).manual_seed(M + 3 * N + 7 * K)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)
    bias = torch.randn(N, device=DEV, generator=g)

    def run():
        out = torch.full((M, N), 7.0, device=DEV, dtype=torch.bfloat16)
        mask = torch.full(((N + 31) // 32, M), -1, device=DEV, dtype=torch.int32)
        gemm_nt(a, b, bias=bias, act="relu", out=out, relu_mask=mask)
        return out, mask

    (o4, m4), (o, m) = _both(monkeypatch, run)
    assert _same(o, o4) and torch.equal(m, m4)


@pytest.mark.parametrize("M,N,K", [(16384, 1536, 960), (1000, 200, 136)])
def test_forward_silu_preact(monkeypatch, M, N, K):
    """5-stage ring: the pre-activation boxes take the second 16 KB of the epilogue area"""
    from pulse_b200.dense import gemm_nt
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)
    bias = torch.randn(N, device=DEV, generator=g)

    def run():
        out = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
        pre = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
        gemm_nt(a, b, bias=bias, act="silu", out=out, preact=pre)
        return out, pre

    (o4, p4), (o, p) = _both(monkeypatch, run)
    assert _same(o, o4) and _same(p, p4)


# (M, N, K) of dgrad: dX [M, N] = dY [M, K] . W [K, N] (W read MN-major)
DGRAD = [(16384, 1024, 512), (12288, 1024, 512), (4096, 1024, 512), (1000, 200, 136)]


@pytest.mark.parametrize("M,N,K", DGRAD)
def test_dgrad_mask_word_gate(monkeypatch, M, N, K):
    from pulse_b200.dense import gemm
    g = torch.Generator(device=DEV).manual_seed(M + 5 * N + K)
    dy, w = _bf(g, M, K), _bf(g, K, N, K ** -0.5)
    words = torch.randint(-2 ** 31, 2 ** 31 - 1, ((N + 31) // 32, M), device=DEV, dtype=torch.int32, generator=g)

    def run():
        out = torch.full((M, N), 7.0, device=DEV, dtype=torch.bfloat16)
        gemm(dy, w, b_mn=True, out=out, gate_mask=words)
        return out

    o4, o = _both(monkeypatch, run)
    assert _same(o, o4)


def test_gradient_penalty_dgrad_alpha_sumsq(monkeypatch):
    """the gradient penalty's G = alpha dY W with its sum of squares (M4096 N1960 K1024)"""
    from pulse_b200.dense import gemm
    M, N, K = 4096, 1960, 1024
    g = torch.Generator(device=DEV).manual_seed(17)
    dy, w = _bf(g, M, K), _bf(g, K, N, K ** -0.5)

    def run():
        out = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
        ss = torch.zeros(1, device=DEV, dtype=torch.float64)
        gemm(dy, w, b_mn=True, out=out, alpha=0.01, sumsq=ss)
        return out, ss

    (o4, s4), (o, s) = _both(monkeypatch, run)
    assert _same(o, o4)
    assert abs(float(s) - float(s4)) <= 1e-12 * float(s4)


def test_strided_output_window(monkeypatch):
    """a GEMM writing into columns [0, 256) of a wider operand (the sept encoder's top layer writes into the policy input)"""
    from pulse_b200.dense import gemm_nt
    M, N, K = 4096, 256, 1088
    g = torch.Generator(device=DEV).manual_seed(11)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)

    def run():
        P = torch.full((M, 640), 3.0, device=DEV, dtype=torch.bfloat16)
        pre = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
        gemm_nt(a, b, act="relu", out=P[:, :N], preact=pre)
        return P, pre

    (P4, p4), (P, p) = _both(monkeypatch, run)
    assert _same(P, P4) and _same(p, p4)
    assert bool((P[:, N:] == 3.0).all())


# (M, N, K) of the weight gradients dW [M, N] += dY^T [M, K] X [K, N] (both MN-major), split-K as the nets pick it: fp32 slabs written by the
# register-resident epilogue, then added in slice order.  N = 934 is not a multiple of 4 and keeps the staged epilogue.
WGRAD = [(1024, 960, 16384), (512, 1024, 16384), (69, 512, 16384), (512, 1024, 4096), (1000, 200, 4096), (1024, 934, 16384)]


@pytest.mark.parametrize("M,N,K", WGRAD)
def test_wgrad_split_k_slabs(monkeypatch, M, N, K):
    from pulse_b200.dense import gemm
    from pulse_b200.nets import pick_split
    g = torch.Generator(device=DEV).manual_seed(M + 7 * N + K)
    dy, x = _bf(g, K, M), _bf(g, K, N)
    split = pick_split(((M + 127) // 128) * ((N + 127) // 128), (K + 63) // 64)
    init = torch.randn(M, N + 4, device=DEV, generator=g)

    def run():
        out = init.clone()
        gemm(dy, x, a_mn=True, b_mn=True, out_f32=out[:, :N], accumulate=True, split_k=split)
        return out

    o4, o = _both(monkeypatch, run)
    assert torch.equal(o, o4)
