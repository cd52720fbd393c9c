"""The bounds of tests/fp64_ref.py have teeth (no GPU needed).

A CPU simulation of each kernel -- bf16 operands, fp32 accumulation over 64-wide k-blocks, the kernel's fp32 epilogue and bf16
roundings -- must pass its comparator, and each mutation below must be rejected by it.  A mutation the bound cannot reject means the
bound is too loose for tests/test_gpu_update_fp64.py to be worth running.
"""
import math

import pytest
import torch

from tests.fp64_ref import BoundError, Gemm, adam_ref, kernel_gemm, check, check_mask, disc_loss_ref, pack_mask, ppo_loss_ref, unpack_mask

BF = torch.bfloat16
_kernel_gemm = kernel_gemm


def _bf(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(BF)


def _setup(seed=0, M=96, K=512, N=256):
    g = torch.Generator().manual_seed(seed)
    return g, _bf(g, M, K), _bf(g, K, N, scale=K ** -0.5)


# ---------------------------------------------------------------------------------------------------- the simulated kernels pass
def test_simulated_forward_relu_mask_and_bf16_output_pass():
    g, a, b = _setup()
    y = _kernel_gemm(a, b)
    ref = Gemm(a, b)
    ref.check(None, "fp32 out", y)
    ref.check(None, "bf16 out", y.to(BF))
    check(None, "relu act", torch.relu(y).to(BF), torch.relu(ref.y), ref.tol(True))
    words = pack_mask(y > 0)
    assert torch.equal(unpack_mask(words, 256, 96), y > 0)
    check_mask(None, "mask", words, ref, 256, 96)


def test_simulated_augmented_input_tail_and_split_k_pass():
    g = torch.Generator().manual_seed(1)
    x = torch.zeros(64, 960, dtype=BF)
    x[:, :934] = _bf(g, 64, 934)
    x[:, 934] = 1.0
    w = torch.zeros(960, 128, dtype=BF)
    w[:935] = _bf(g, 935, 128, scale=0.05)
    Gemm(x, w).check(None, "aug forward", _kernel_gemm(x, w).to(BF))
    dy, xin = _bf(g, 1000, 64), _bf(g, 1000, 72)
    Gemm(dy.T, xin).check(None, "wgrad split-K", _kernel_gemm(dy.T, xin, slices=4))


def test_simulated_adam_passes():
    g = torch.Generator().manual_seed(2)
    n = 4096
    p, grad = torch.randn(n, generator=g) * 0.05, torch.randn(n, generator=g) * 1e-3
    m, v = torch.randn(n, generator=g) * 1e-4, torch.rand(n, generator=g) * 1e-6
    grad[:64] = 0.0
    m[:64], v[:64] = 0.0, 0.0
    for max_norm in (1e9, 0.5 * float(grad.norm())):
        p1, m1, v1 = _kernel_adam(p, grad, m, v, step=2, lr=2e-5, max_norm=max_norm)
        rp, rm, rv, dp, dm, dv, clipped, _ = adam_ref(p, grad, m, v, 2, lr=2e-5, max_norm=max_norm)
        assert clipped == (max_norm < 1e8)
        check(None, "p", p1, rp, dp)
        check(None, "m", m1, rm, dm)
        check(None, "v", v1, rv, dv)


def _kernel_adam(p, g, m, v, step, lr, max_norm, b1=0.9, b2=0.999, eps=1e-8, bias_step=None, clip=True):
    """pulse_adam_step's fp32 arithmetic (csrc/mlp_ops.cu adam_kernel)."""
    f = lambda x: torch.tensor(x, dtype=torch.float32)
    t = f(float(step + 1 if bias_step is None else bias_step))
    b1f, b2f, lrf, epsf = f(b1), f(b2), f(lr), f(eps)
    bc1, bc2 = 1 - torch.pow(b1f, t), 1 - torch.pow(b2f, t)
    scale = f(1.0)
    if clip and max_norm > 0:
        norm = f(float(torch.sqrt((g.double() ** 2).sum())))
        scale = torch.clamp(f(max_norm) / (norm + f(1e-6)), max=1.0)
    gi = g * scale
    m1 = b1f * m + (1 - b1f) * gi
    v1 = b2f * v + (1 - b2f) * gi * gi
    p1 = p - (lrf / bc1) * m1 / (torch.sqrt(v1) / torch.sqrt(bc2) + epsf)
    return p1, m1, v1


def _kernel_ppo(mu, value, actions, old_nlp, adv, ret, logstd, e_clip=0.2, critic_coef=5.0, bounds_coef=10.0):
    """pulse_ppo_loss's fp32 arithmetic: dmu / dv in bf16."""
    M, A = mu.shape
    sg = torch.exp(logstd)
    z = (actions - mu) / sg
    nlp = 0.5 * (z * z).sum(-1) + 0.5 * 1.8378770664093453 * A + logstd.sum()
    ratio = torch.exp(old_nlp - nlp)
    rc = torch.clamp(ratio, 1 - e_clip, 1 + e_clip)
    s1, s2 = -adv * ratio, -adv * rc
    da = torch.where(s1 >= s2, adv * ratio, torch.zeros_like(ratio))
    hi, lo = torch.clamp_min(mu - 1, 0), torch.clamp_max(mu + 1, 0)
    g = (da[:, None] * (-(actions - mu) / (sg * sg)) + bounds_coef * 2 * (hi + lo)) * (1.0 / M)
    dv = -2 * (ret - value) * critic_coef * (1.0 / M)
    return g.to(BF), dv.to(BF)


def _ppo_inputs(seed=3, M=512, A=69):
    g = torch.Generator().manual_seed(seed)
    logstd = torch.full((A,), -2.9)
    mu = torch.randn(M, A, generator=g) * 0.5
    mu[:, :4] += torch.tensor([1.5, -1.5, 1.2, -1.2])
    actions = mu + torch.exp(logstd) * torch.randn(M, A, generator=g)
    z = (actions - mu) / torch.exp(logstd)
    nlp = 0.5 * (z * z).sum(-1) + 0.5 * math.log(2 * math.pi) * A + logstd.sum()
    grp = torch.arange(M) % 4
    old = nlp + torch.where(grp == 1, 0.4, torch.where(grp == 2, -0.4, torch.where(grp == 3, 0.4, 0.0)))
    adv = torch.randn(M, generator=g)
    adv = torch.where(grp == 1, adv.abs() + 0.1, torch.where(grp >= 2, -(adv.abs() + 0.1), adv))
    return mu, torch.randn(M, generator=g), actions, old, adv, torch.randn(M, generator=g), logstd


def test_simulated_ppo_loss_passes():
    mu, value, actions, old, adv, ret, logstd = _ppo_inputs()
    dmu, dv = _kernel_ppo(mu, value, actions, old, adv, ret, logstd)
    ref = ppo_loss_ref(mu, value, actions, old, adv, ret, logstd)
    tol = torch.where(ref["ambiguous"][:, None], torch.full_like(ref["tol_mu"], math.inf), ref["tol_mu"])
    assert int(ref["ambiguous"].sum()) <= 2
    check(None, "dmu", dmu, ref["dmu"], tol)
    check(None, "dv", dv, ref["dv"], ref["tol_v"])


def test_simulated_disc_loss_passes():
    g = torch.Generator().manual_seed(4)
    l = torch.randn(300, generator=g) * 3
    sg = torch.sigmoid(l)
    d = torch.where(torch.arange(300) < 200, 0.5 * 5.0 * sg / 200, 0.5 * 5.0 * (sg - 1) / 100).to(BF)
    ref, tol, _, _ = disc_loss_ref(l, 200, 5.0)
    check(None, "dlogit", d, ref, tol)


# --------------------------------------------------------------------------------------------------------- mutations are rejected
def _rejects(fn):
    with pytest.raises(BoundError):
        fn()


def test_rejects_missing_k_block_in_one_tile():
    g, a, b = _setup()
    y = _kernel_gemm(a, b, skip=(3, slice(128, 256)))
    _rejects(lambda: Gemm(a, b).check(None, "fp32", y))
    _rejects(lambda: Gemm(a, b).check(None, "bf16", y.to(BF)))


def test_rejects_dropped_k_tail_of_the_69_wide_head():
    g = torch.Generator().manual_seed(5)
    dmu, w = _bf(g, 256, 69, scale=1e-3), _bf(g, 69, 512, scale=0.05)           # actor head dgrad: K = 69 actions
    good = _kernel_gemm(dmu, w)
    Gemm(dmu, w).check(None, "head dgrad", good.to(BF))
    _rejects(lambda: Gemm(dmu, w).check(None, "head dgrad", _kernel_gemm(dmu[:, :64], w[:64]).to(BF)))


def test_rejects_dropped_k_tail_of_the_935_wide_input():
    g = torch.Generator().manual_seed(6)
    x = torch.zeros(64, 960, dtype=BF)
    x[:, :934] = _bf(g, 64, 934)
    x[:, 934] = 1.0
    w = torch.zeros(960, 128, dtype=BF)
    w[:935] = _bf(g, 935, 128, scale=0.05)
    _rejects(lambda: Gemm(x, w).check(None, "layer 0", _kernel_gemm(x[:, :896], w[:896]).to(BF)))


def test_rejects_split_k_slice_counted_twice():
    g = torch.Generator().manual_seed(7)
    dy, xin = _bf(g, 1000, 64), _bf(g, 1000, 72)
    _rejects(lambda: Gemm(dy.T, xin).check(None, "wgrad", _kernel_gemm(dy.T, xin, slices=4, dup_slice=2)))


def test_rejects_ones_column_omitted():
    g = torch.Generator().manual_seed(8)
    x = torch.zeros(64, 960, dtype=BF)
    x[:, :934] = _bf(g, 64, 934)
    x[:, 934] = 1.0
    w = torch.zeros(960, 128, dtype=BF)
    w[:935] = _bf(g, 935, 128, scale=0.05)
    x0 = x.clone()
    x0[:, 934] = 0.0
    _rejects(lambda: Gemm(x, w).check(None, "aug forward", _kernel_gemm(x0, w).to(BF)))


def test_rejects_bias_omitted():
    g, a, b = _setup(9)
    bias = torch.randn(256, generator=g) * 0.05
    _rejects(lambda: Gemm(a, b, bias=bias).check(None, "plain forward", _kernel_gemm(a, b).to(BF)))


def test_rejects_mask_words_shifted_by_one_column():
    g, a, b = _setup(10)
    y = _kernel_gemm(a, b)
    words = pack_mask(y > 0)
    check_mask(None, "mask", words, Gemm(a, b), 256, 96)
    bad = words.clone()
    bad[1] = bad[1] << 1                                  # columns 32..63 read one column off
    _rejects(lambda: check_mask(None, "mask", bad, Gemm(a, b), 256, 96))


def test_rejects_gate_from_agent_rows():
    """g1 = m1 * (g2 W2) on the demo rows; the mutant gates with the agent rows' masks (rows [0, B) of the 3B-row workspace)."""
    g = torch.Generator().manual_seed(11)
    B = 64
    masks = torch.randn(3 * B, 128, generator=g) > 0
    m_agent, m_demo = masks[:B], masks[2 * B:]
    g2, w2 = _bf(g, B, 96), _bf(g, 96, 128, scale=0.1)
    wrong = (_kernel_gemm(g2, w2) * m_agent).to(BF)
    Gemm(g2, w2, gate=m_demo).check(None, "g1", (_kernel_gemm(g2, w2) * m_demo).to(BF))
    _rejects(lambda: Gemm(g2, w2, gate=m_demo).check(None, "g1", wrong))


def test_rejects_gradient_penalty_coefficient_off_by_one_percent():
    g = torch.Generator().manual_seed(12)
    g1, w1 = _bf(g, 64, 256), _bf(g, 256, 192, scale=0.05)
    c = 2.0 * 5.0 * 5.0 / 64
    good = (_kernel_gemm(g1, w1) * c).to(BF)
    Gemm(g1, w1, alpha=c).check(None, "G", good)
    _rejects(lambda: Gemm(g1, w1, alpha=c).check(None, "G", (_kernel_gemm(g1, w1) * (c * 1.01)).to(BF)))


def _adam_case():
    g = torch.Generator().manual_seed(13)
    n = 4096
    return (torch.randn(n, generator=g) * 0.05, torch.randn(n, generator=g) * 1e-3, torch.randn(n, generator=g) * 1e-4,
            torch.rand(n, generator=g) * 1e-6)


def test_rejects_adam_bias_correction_of_the_previous_step():
    p, grad, m, v = _adam_case()
    rp, rm, rv, dp, dm, dv, _, _ = adam_ref(p, grad, m, v, 2, lr=2e-5, max_norm=1e9)
    p1, _, _ = _kernel_adam(p, grad, m, v, step=2, lr=2e-5, max_norm=1e9, bias_step=2)     # t - 1 instead of t = 3
    _rejects(lambda: check(None, "p", p1, rp, dp))


def test_rejects_adam_ignoring_the_clip():
    p, grad, m, v = _adam_case()
    max_norm = 0.5 * float(grad.norm())
    rp, rm, rv, dp, dm, dv, clipped, _ = adam_ref(p, grad, m, v, 2, lr=2e-5, max_norm=max_norm)
    assert clipped
    p1, m1, v1 = _kernel_adam(p, grad, m, v, step=2, lr=2e-5, max_norm=max_norm, clip=False)

    def all_three():
        check(None, "p", p1, rp, dp)
        check(None, "m", m1, rm, dm)
        check(None, "v", v1, rv, dv)
    _rejects(all_three)
    _rejects(lambda: check(None, "m", m1, rm, dm))
