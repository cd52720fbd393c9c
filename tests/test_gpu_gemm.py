"""wgmma bf16 GEMM vs a plain PyTorch fp32 reference of the same op (bf16-rounded inputs)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, bias=None, act=None, alpha=1.0):
    y = alpha * (a.float() @ b.float().T)
    if bias is not None:
        y = y + bias
    pre = y
    if act == "relu":
        y = torch.relu(y)
    elif act == "silu":
        y = torch.nn.functional.silu(y)
    return y, pre


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 384, 960), (300, 200, 136), (128, 128, 1024), (16384, 1024, 960), (77, 69, 512)])
def test_gemm_fp32_and_bf16_outputs(M, N, K):
    from pulse_b200.dense import gemm_nt
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device=dev, generator=g).bfloat16()
    b = (torch.randn(N, K, device=dev, generator=g) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device=dev, generator=g)
    of = torch.full((M, N), float("nan"), device=dev)
    ob = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    gemm_nt(a, b, bias=bias, act="relu", out=ob, out_f32=of)
    torch.cuda.synchronize()
    ref, _ = _ref(a, b, bias, "relu")
    torch.testing.assert_close(of, ref, atol=2e-3, rtol=2e-3)
    torch.testing.assert_close(ob.float(), ref, atol=2e-2, rtol=2e-2)


def test_gemm_epilogue_variants():
    from pulse_b200.dense import gemm_nt
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(5)
    M, N, K = 384, 264, 200
    a = torch.randn(M, 208, device=dev, generator=g).bfloat16()[:, :K]     # lda 208 > K
    b = (torch.randn(N, 256, device=dev, generator=g) / K ** 0.5).bfloat16()[:, :K]
    bias = torch.randn(N, device=dev, generator=g)
    out = torch.zeros(M, 272, device=dev, dtype=torch.bfloat16)[:, :N]
    out_t = torch.zeros(N, M, device=dev, dtype=torch.bfloat16)
    pre = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    gemm_nt(a, b, bias=bias, act="silu", out=out, out_t=out_t, preact=pre, alpha=0.5)
    ref, refpre = _ref(a, b, bias, "silu", alpha=0.5)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(out_t.float(), ref.T, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(pre.float(), refpre, atol=2e-2, rtol=2e-2)
    # backward-style gating: result * relu'(saved output) and * silu'(saved pre-activation)
    gate = torch.randn(M, N, device=dev, generator=g).bfloat16()
    of = torch.zeros(M, N, device=dev)
    gemm_nt(a, b, gate=gate, gate_mode="relu", out_f32=of)
    torch.testing.assert_close(of, _ref(a, b)[0] * (gate.float() > 0), atol=2e-3, rtol=2e-3)
    gemm_nt(a, b, gate=gate, gate_mode="silu", out_f32=of)
    z = gate.float()
    s = torch.sigmoid(z)
    torch.testing.assert_close(of, _ref(a, b)[0] * (s * (1 + z * (1 - s))), atol=2e-3, rtol=2e-3)


def test_gemm_split_k_slabs():
    from pulse_b200.dense import gemm_nt, num_splits
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(9)
    M, N, K = 256, 192, 4096 + 64
    a = torch.randn(M, K, device=dev, generator=g).bfloat16()
    b = (torch.randn(N, K, device=dev, generator=g) / K ** 0.5).bfloat16()
    ns = num_splits(K, 6)
    slabs = torch.zeros(ns, M, N, device=dev)
    gemm_nt(a, b, out_f32=slabs, split_k=6)
    torch.testing.assert_close(slabs.sum(0), _ref(a, b)[0], atol=3e-3, rtol=3e-3)


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(256, 384, 960), (300, 200, 136), (1024, 960, 16384), (69, 512, 4096)])
def test_gemm_mn_major_operands(a_mn, b_mn, M, N, K):
    """dgrad / wgrad forms: operands consumed as they sit in memory (reduction index = row index)."""
    from pulse_b200.dense import gemm
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(M + 3 * N + 7 * K + a_mn + 2 * b_mn)
    pad = lambda n: (n + 7) // 8 * 8
    A = torch.randn(M, K, device=dev, generator=g)
    B = torch.randn(N, K, device=dev, generator=g) / K ** 0.5
    a = torch.zeros(K, pad(M), device=dev, dtype=torch.bfloat16)[:, :M] if a_mn else torch.zeros(M, pad(K), device=dev, dtype=torch.bfloat16)[:, :K]
    b = torch.zeros(K, pad(N), device=dev, dtype=torch.bfloat16)[:, :N] if b_mn else torch.zeros(N, pad(K), device=dev, dtype=torch.bfloat16)[:, :K]
    a.copy_(A.T if a_mn else A)
    b.copy_(B.T if b_mn else B)
    ref = (a.float().T if a_mn else a.float()) @ (b.float() if b_mn else b.float().T)
    of = torch.zeros(M, N, device=dev)
    gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=of)
    torch.testing.assert_close(of, ref, atol=3e-3, rtol=3e-3)
    # atomic accumulation across split-K + column sums of the result
    acc = torch.ones(M, N, device=dev)
    gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=acc, accumulate=True, split_k=3)
    torch.testing.assert_close(acc - 1.0, ref, atol=5e-3, rtol=5e-3)
    cs = torch.zeros(N, device=dev)
    ob = torch.zeros(M, pad(N), device=dev, dtype=torch.bfloat16)
    gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=ob, colsum=cs)
    torch.testing.assert_close(cs, ref.sum(0), atol=2e-2 * M ** 0.5, rtol=2e-2)
    torch.testing.assert_close(ob[:, :N].float(), ref, atol=2e-2, rtol=2e-2)


def test_gemm_rejects_bad_arguments():
    from pulse_b200 import PulseError
    from pulse_b200.dense import gemm_nt
    dev = torch.device("cuda:0")
    a = torch.zeros(128, 70, device=dev, dtype=torch.bfloat16)
    b = torch.zeros(128, 70, device=dev, dtype=torch.bfloat16)
    with pytest.raises(PulseError):
        gemm_nt(a, b, out_f32=torch.zeros(128, 128, device=dev))  # lda = 70 not a multiple of 8
    with pytest.raises(PulseError):
        gemm_nt(a[:, :64].contiguous(), b[:, :64].contiguous())      # no output


@pytest.mark.parametrize("M,N,K", [(512, 512, 128), (300, 1000, 72), (4096, 1960, 1024)])
def test_gemm_relu_gate_mask_and_sumsq(M, N, K):
    """Fast ReLU-gate path (128 gate values per thread folded to a bit mask before the accumulator wait) on full and ragged
    128-column groups, including -0.0 / tiny / negative gate values, plus the fused sum-of-squares reduction."""
    from pulse_b200.dense import gemm
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(M + N + K)
    a = torch.randn(M, K, device=dev, generator=g).bfloat16()
    b = (torch.randn(K, N + 8, device=dev, generator=g) / K ** 0.5).bfloat16()[:, :N]     # MN-major B, ld > N
    gate = torch.randn(M, N + 8, device=dev, generator=g)
    gate[::3] = torch.relu(gate[::3])                      # exact +0.0 entries
    gate[1::7, ::5] = -0.0
    gate[2::11, 1::4] = 1e-30                              # flushes to a tiny positive bf16 (still > 0)
    gate = gate.bfloat16()[:, :N]
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    colsum = torch.zeros(N, device=dev)
    sumsq = torch.zeros(2, device=dev, dtype=torch.float64)
    gemm(a, b, b_mn=True, gate=gate, gate_mode="relu", alpha=0.25, out=out, colsum=colsum, sumsq=sumsq)
    ref = 0.25 * (a.float() @ b.float()) * (gate.float() > 0)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(colsum, ref.sum(0), atol=5e-2, rtol=2e-3)
    torch.testing.assert_close(sumsq[0], (ref.double() ** 2).sum(), atol=1e-3, rtol=1e-4)
    assert float(sumsq[1]) == 0.0


@pytest.mark.parametrize("M,N,K", [(512, 512, 128), (300, 1000, 72), (16384, 1024, 512), (5000, 768, 256), (16384, 512, 69)])
def test_gemm_relu_dgrad_gate_and_column_sums(M, N, K):
    """ReLU dgrad as the MLP backward issues it (gate + bias-gradient column sums + bf16 output, no sumsq): several tiles per
    CTA, column-tile counts that do and do not divide the grid, ragged edges, the K = 69 actor-head shape."""
    from pulse_b200.dense import gemm
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(7 * M + N + K)
    a = torch.randn(M, (K + 7) // 8 * 8, device=dev, generator=g).bfloat16()[:, :K]      # 16-byte row pitch (K = 69 -> ld 72), as the MLP buffers
    b = (torch.randn(K, N + 8, device=dev, generator=g) / K ** 0.5).bfloat16()[:, :N]
    gate = torch.randn(M, N + 8, device=dev, generator=g)
    gate[::3] = torch.relu(gate[::3])
    gate[1::7, ::5] = -0.0
    gate = gate.bfloat16()[:, :N]
    out = torch.full((M, N), 7.0, device=dev, dtype=torch.bfloat16)
    colsum = torch.zeros(N, device=dev)
    gemm(a, b, b_mn=True, gate=gate, gate_mode="relu", out=out, colsum=colsum)
    ref = (a.float() @ b.float()) * (gate.float() > 0)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(colsum, ref.sum(0), atol=0.25 + 4e-3 * M ** 0.5, rtol=5e-3)
    torch.testing.assert_close(colsum, out.float().sum(0), atol=0.25 + 4e-3 * M ** 0.5, rtol=5e-3)
