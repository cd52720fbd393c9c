"""The 128 x 256 GEMM tile against the 128 x 128 one (PULSE_GEMM_BN=128): each output element runs the same k16 steps in the same order
and the same epilogue arithmetic, so outputs and mask words must match bit for bit.  The fp64 sum of squares takes the same fp32 terms
from both kernels (one per warp and 128 columns), but its atomics land in scheduling order, so it may differ in its last bits.
Every case also checks the tile width each launch took: 128 with PULSE_GEMM_BN=128, the expected width (on an H100's 132 SMs)
without."""
import pytest
import torch

from pulse_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _bf(g, r, c, scale=1.0):
    """bf16 [r, c] view with rows padded to 16 bytes (the GEMM's operand alignment)"""
    return (torch.randn(r, (c + 7) // 8 * 8, device=DEV, generator=g) * scale).bfloat16()[:, :c]


def _both(monkeypatch, run, wide):
    """run() (one GEMM launch) with the narrow tile forced, then with the shape rule; returns both results.  wide: the default launch
    must take the 128 x 256 tile (checked on 132 SMs, the count the shape expectations are written for)"""
    monkeypatch.setenv("PULSE_GEMM_BN", "128")
    ref = run()
    assert _lib.gemm_last_launch()["tile_n"] == 128
    monkeypatch.delenv("PULSE_GEMM_BN")
    new = run()
    if torch.cuda.get_device_properties(DEV).multi_processor_count == 132:
        assert _lib.gemm_last_launch()["tile_n"] == (256 if wide else 128)
    torch.cuda.synchronize()
    return ref, new


def _same(x: torch.Tensor, y: torch.Tensor) -> bool:
    return torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x, y.view(torch.int16) if y.dtype == torch.bfloat16 else y)


# (M, N, K, wide on an H100's 132 SMs): the update's forward shapes (actor / critic at 16384 rows, the discriminator at 12288), N = 1960
# (not a multiple of 256), wide row tails (M = 8000: the last tile's second warpgroup has no rows); at M = 1000 the narrow items fit one
# round, so N = 1960, 934 (not a multiple of 8, staged epilogue) and 200 keep the narrow tile
FWD = [(16384, 1024, 960, True), (16384, 512, 1024, True), (12288, 1024, 1984, True), (12288, 512, 1024, False), (4096, 1960, 1024, True),
       (8000, 1024, 960, True), (8000, 1960, 1000, True), (1000, 1960, 960, False), (1000, 934, 960, False), (1000, 200, 136, False)]


@pytest.mark.parametrize("M,N,K,wide", FWD)
def test_forward_relu_mask_words(monkeypatch, M, N, K, wide):
    from pulse_b200.dense import gemm_nt
    g = torch.Generator(device=DEV).manual_seed(M + 3 * N + 7 * K)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)

    def run():
        out = torch.full((M, N), 7.0, device=DEV, dtype=torch.bfloat16)
        mask = torch.full(((N + 31) // 32, M), -1, device=DEV, dtype=torch.int32)
        gemm_nt(a, b, act="relu", out=out, relu_mask=mask)
        return out, mask

    (o4, m4), (o, m) = _both(monkeypatch, run, wide)
    assert _same(o, o4) and torch.equal(m, m4)


@pytest.mark.parametrize("M,N,K", [(16384, 1024, 960), (8000, 1960, 1024)])
def test_forward_bias(monkeypatch, M, N, K):
    """the wide epilogue reads the bias from global memory, the narrow one from its shared copy"""
    from pulse_b200.dense import gemm_nt
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)
    bias = torch.randn(N, device=DEV, generator=g)

    def run():
        out = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
        gemm_nt(a, b, bias=bias, act="relu", out=out)
        return out

    o4, o = _both(monkeypatch, run, True)
    assert _same(o, o4)


# (M, N, K) of dgrad: dX [M, N] = dY [M, K] . W [K, N] (W read MN-major), gated by mask words: the update's layer-1 dgrad at 16384 and
# 12288 rows, the gradient penalty's g1 at 4096, a row tail with N = 1960; the K = 69 head dgrad keeps the narrow tile
DGRAD = [(16384, 1024, 512, True), (12288, 1024, 512, True), (4096, 1024, 512, True), (8000, 1960, 512, True), (16384, 512, 69, False)]


@pytest.mark.parametrize("M,N,K,wide", DGRAD)
def test_dgrad_mask_word_gate(monkeypatch, M, N, K, wide):
    from pulse_b200.dense import gemm
    g = torch.Generator(device=DEV).manual_seed(M + 5 * N + K)
    dy, w = _bf(g, M, K), _bf(g, K, N, K ** -0.5)
    words = torch.randint(-2 ** 31, 2 ** 31 - 1, ((N + 31) // 32, M), device=DEV, dtype=torch.int32, generator=g)

    def run():
        out = torch.full((M, N), 7.0, device=DEV, dtype=torch.bfloat16)
        gemm(dy, w, b_mn=True, out=out, gate_mask=words)
        return out

    o4, o = _both(monkeypatch, run, wide)
    assert _same(o, o4)


def test_dgrad_k_major_b(monkeypatch):
    """the gradient penalty's du = m1 * (G W1^T): both operands K-major, so the wide B stage is one 256-row box"""
    from pulse_b200.dense import gemm
    M, N, K = 4096, 1024, 1960
    g = torch.Generator(device=DEV).manual_seed(23)
    G, w = _bf(g, M, K), _bf(g, N, K, K ** -0.5)
    words = torch.randint(-2 ** 31, 2 ** 31 - 1, ((N + 31) // 32, M), device=DEV, dtype=torch.int32, generator=g)

    def run():
        out = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
        gemm(G, w, gate_mask=words, out=out)
        return out

    o4, o = _both(monkeypatch, run, True)
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

    (o4, s4), (o, s) = _both(monkeypatch, run, True)
    assert _same(o, o4)
    assert abs(float(s) - float(s4)) <= 1e-12 * float(s4)


def test_strided_output_window(monkeypatch):
    """a wide GEMM writing into columns [0, 512) of a wider buffer: the columns beyond stay untouched"""
    from pulse_b200.dense import gemm_nt
    M, N, K = 16384, 512, 1024
    g = torch.Generator(device=DEV).manual_seed(11)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)

    def run():
        P = torch.full((M, 1280), 3.0, device=DEV, dtype=torch.bfloat16)
        mask = torch.zeros(N // 32, M, device=DEV, dtype=torch.int32)
        gemm_nt(a, b, act="relu", out=P[:, :N], relu_mask=mask)
        return P, mask

    (P4, m4), (P, m) = _both(monkeypatch, run, True)
    assert _same(P, P4) and torch.equal(m, m4)
    assert bool((P[:, N:] == 3.0).all())
