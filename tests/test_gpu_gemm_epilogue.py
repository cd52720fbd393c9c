"""The register-resident GEMM epilogue (bf16 outputs, ReLU mask words, mask-word gate, sum of squares) against the staged fp32
epilogue of the same GEMM: the fp32 values are the same, so the bf16 outputs and mask words must match bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _bf(g, r, c, scale=1.0):
    """bf16 [r, c] view with rows padded to 16 bytes (the GEMM's operand alignment)"""
    return (torch.randn(r, (c + 7) // 8 * 8, device=DEV, generator=g) * scale).bfloat16()[:, :c]


def _mask_words(pos: torch.Tensor) -> torch.Tensor:
    """[M, N] bool -> int64 [ceil(N/32), M] words, bit i of word c = column 32 c + i"""
    M, N = pos.shape
    C = (N + 31) // 32
    p = torch.zeros(M, C * 32, dtype=torch.int64, device=pos.device)
    p[:, :N] = pos.long()
    w = (p.view(M, C, 32) << torch.arange(32, device=pos.device)).sum(-1)
    return w.t().contiguous()


def _words(t: torch.Tensor) -> torch.Tensor:
    return t.long() & 0xFFFFFFFF


def _same(x: torch.Tensor, y: torch.Tensor) -> bool:
    return torch.equal(x.float(), y.float())


# (M, N, K): the update shapes, row tails (4096 / 1000), column tails (200; N = 69 is not a whole number of 16-byte units and takes
# the staged path)
FWD = [(16384, 1024, 960), (16384, 512, 1024), (12288, 1024, 1984), (4096, 1024, 1960), (1000, 512, 960), (4096, 69, 512), (1000, 200, 136)]


@pytest.mark.parametrize("M,N,K", FWD)
@pytest.mark.parametrize("with_bias", [False, True])
def test_forward_relu_matches_staged(M, N, K, with_bias):
    from pulse_b200.dense import gemm_nt
    g = torch.Generator(device=DEV).manual_seed(M + 3 * N + 7 * K + with_bias)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)
    bias = torch.randn(N, device=DEV, generator=g) if with_bias else None
    ld = (N + 63) // 64 * 64 + 64                       # wider rows: columns >= N must stay untouched
    f32 = torch.zeros(M, N, device=DEV)
    gemm_nt(a, b, bias=bias, out_f32=f32)               # staged path: the fp32 pre-activation
    out = torch.full((M, ld), 7.0, device=DEV, dtype=torch.bfloat16)
    pre = torch.full((M, ld), 7.0, device=DEV, dtype=torch.bfloat16)
    mask = torch.full(((N + 31) // 32, M + 8), -1, device=DEV, dtype=torch.int32)
    gemm_nt(a, b, bias=bias, act="relu", out=out, preact=pre, relu_mask=mask)
    torch.cuda.synchronize()
    assert _same(pre[:, :N], f32.bfloat16())
    assert _same(out[:, :N], torch.relu(f32).bfloat16())
    assert torch.equal(_words(mask[:, :M]), _mask_words(f32 > 0))
    assert bool((out[:, N:] == 7.0).all()) and bool((pre[:, N:] == 7.0).all()) and bool((mask[:, M:] == -1).all())


@pytest.mark.parametrize("M,N,K", [(16384, 1536, 960), (1000, 200, 136), (4096, 160, 512)])
def test_forward_silu_matches_staged(M, N, K):
    from pulse_b200.dense import gemm_nt
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)
    bias = torch.randn(N, device=DEV, generator=g)
    f32 = torch.zeros(M, N, device=DEV)
    gemm_nt(a, b, bias=bias, out_f32=f32)
    out = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    pre = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    gemm_nt(a, b, bias=bias, act="silu", out=out, preact=pre)
    torch.cuda.synchronize()
    assert _same(pre, f32.bfloat16())
    # SiLU runs on fast-math exp / divide: within one bf16 rounding of the exact value
    torch.testing.assert_close(out.float(), torch.nn.functional.silu(pre.float()), atol=1e-2, rtol=1e-2)


# (M, N, K) of dgrad: dX [M, N] = dY [M, K] . W [K, N] (W read MN-major)
DGRAD = [(16384, 1024, 512), (12288, 1024, 512), (4096, 1024, 512), (4096, 1960, 1024), (1000, 512, 69), (4096, 69, 512), (1000, 200, 136)]


@pytest.mark.parametrize("M,N,K", DGRAD)
@pytest.mark.parametrize("gated", [False, True])
def test_dgrad_matches_staged(M, N, K, gated):
    from pulse_b200.dense import gemm
    g = torch.Generator(device=DEV).manual_seed(M + 5 * N + K + gated)
    dy, w = _bf(g, M, K), _bf(g, K, N, K ** -0.5)
    alpha = 1.0 if gated else 0.37
    kw = dict(b_mn=True, alpha=alpha)
    if gated:   # a [C, >= M] view with a longer row stride, like the gradient penalty's demo rows
        words = torch.randint(-2 ** 31, 2 ** 31 - 1, ((N + 31) // 32, 3 * M), device=DEV, dtype=torch.int32, generator=g)
        kw["gate_mask"] = words[:, 2 * M:]
    f32 = torch.zeros(M, N, device=DEV)
    gemm(dy, w, out_f32=f32, **kw)                      # staged path: gated fp32
    ld = (N + 63) // 64 * 64
    out = torch.full((M, ld), 7.0, device=DEV, dtype=torch.bfloat16)
    ss = torch.zeros(1, device=DEV, dtype=torch.float64)
    gemm(dy, w, out=out, sumsq=ss, **kw)
    torch.cuda.synchronize()
    if gated:   # the staged reference did apply the gate
        sel = ((_words(kw["gate_mask"]).t().unsqueeze(-1) >> torch.arange(32, device=DEV)) & 1).reshape(M, -1)[:, :N].bool()
        assert bool((f32[~sel] == 0).all())
    assert _same(out[:, :N], f32.bfloat16())
    assert bool((out[:, N:] == 7.0).all())
    ref = (f32.double() ** 2).sum()
    assert abs(float(ss) - float(ref)) <= 1e-5 * float(ref)


def test_strided_output_window():
    """A GEMM writing into columns [0, 256) of a wider operand (the sept encoder's top layer writes into the policy input)."""
    from pulse_b200.dense import gemm_nt
    M, N, K = 4096, 256, 1088
    g = torch.Generator(device=DEV).manual_seed(11)
    a, b = _bf(g, M, K), _bf(g, N, K, K ** -0.5)
    P = torch.full((M, 640), 3.0, device=DEV, dtype=torch.bfloat16)
    pre = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16)
    f32 = torch.zeros(M, N, device=DEV)
    gemm_nt(a, b, out_f32=f32)
    gemm_nt(a, b, act="relu", out=P[:, :N], preact=pre)
    torch.cuda.synchronize()
    assert _same(P[:, :N], torch.relu(f32).bfloat16())
    assert _same(pre, f32.bfloat16())
    assert bool((P[:, N:] == 3.0).all())
