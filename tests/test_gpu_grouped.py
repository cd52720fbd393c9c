"""Grouped GEMM launches (several problems per persistent launch) and the lock-step actor + critic update built on them (the
product path does not use grouped launches unless PULSE_GROUPED=1)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bf(*shape, gen, scale=1.0):
    return (torch.randn(*shape, device=DEV, generator=gen) * scale).bfloat16()


def test_grouped_forward_matches_single_launches():
    from pulse_b200.dense import gemm, gemm_grouped
    g = torch.Generator(device=DEV).manual_seed(1)
    probs, refs = [], []
    for (M, N, K) in ((2048, 1024, 960), (2048, 512, 1024), (700, 300, 72), (4096, 1536, 384)):
        a, w, bias = _bf(M, K, gen=g), _bf(N, K, gen=g, scale=K ** -0.5), torch.randn(N, device=DEV, generator=g)
        out1 = torch.zeros(M, (N + 7) // 8 * 8, device=DEV, dtype=torch.bfloat16)
        out2 = torch.zeros_like(out1)
        gemm(a, w, bias=bias, act="relu", out=out1)
        probs.append((a, w, dict(bias=bias, act="relu", out=out2)))
        refs.append((out1, out2))
    gemm_grouped(probs)
    for out1, out2 in refs:
        assert torch.equal(out1, out2)


def test_grouped_wgrad_and_dgrad_match_single_launches():
    from pulse_b200.dense import gemm, gemm_grouped
    from pulse_b200.nets import pick_split
    g = torch.Generator(device=DEV).manual_seed(2)
    wg, dg, checks = [], [], []
    for (M, N, K) in ((4096, 1024, 960), (4096, 512, 1024)):           # batch M, layer N x K
        dy, x, w = _bf(M, N, gen=g, scale=0.1), _bf(M, K, gen=g), _bf(N, K, gen=g, scale=K ** -0.5)
        gate = torch.relu(_bf(M, K, gen=g))
        dw1, dw2 = torch.zeros(N, K, device=DEV), torch.zeros(N, K, device=DEV)
        sk = pick_split(((N + 127) // 128) * ((K + 255) // 256), (M + 63) // 64)
        gemm(dy, x, a_mn=True, b_mn=True, out_f32=dw1, accumulate=True, split_k=sk)
        wg.append((dy, x, dict(a_mn=True, b_mn=True, out_f32=dw2, accumulate=True, split_k=sk)))
        dx1, dx2 = torch.zeros(M, K, device=DEV, dtype=torch.bfloat16), torch.zeros(M, K, device=DEV, dtype=torch.bfloat16)
        cs1, cs2 = torch.zeros(K, device=DEV), torch.zeros(K, device=DEV)
        gemm(dy, w, b_mn=True, gate=gate, gate_mode="relu", out=dx1, colsum=cs1)
        dg.append((dy, w, dict(b_mn=True, gate=gate, gate_mode="relu", out=dx2, colsum=cs2)))
        checks.append((dw1, dw2, dx1, dx2, cs1, cs2))
    gemm_grouped(wg)
    gemm_grouped(dg)
    for dw1, dw2, dx1, dx2, cs1, cs2 in checks:
        torch.testing.assert_close(dw2, dw1, atol=1e-3, rtol=1e-4)      # fp32 atomics: order differs
        assert torch.equal(dx1, dx2)
        torch.testing.assert_close(cs2, cs1, atol=1e-2, rtol=1e-4)


def test_ppo_minibatch_grouped_matches_three_stream_path(monkeypatch):
    from pulse_b200.ppo import PPOPolicy
    g = torch.Generator(device=DEV).manual_seed(3)
    M = 2048
    obs = torch.randn(M, 934, device=DEV, generator=g)
    # a PPO minibatch as a rollout hands it over: actions drawn by the same policy, old neglogp close to the current one (ratios
    # around 1, some clipped).  Far-off old neglogp overflows exp(old - new) in fp32 and makes both paths' gradients NaN.
    drawn = PPOPolicy(device=DEV, seed=5).act(obs, eps=torch.randn(M, 69, device=DEV, generator=g))
    act = drawn["actions"].clone()
    nlp = drawn["neglogpacs"].clone() + 0.3 * torch.randn(M, device=DEV, generator=g)
    adv, ret = torch.randn(M, device=DEV, generator=g), torch.randn(M, device=DEV, generator=g)
    results = []
    for flag in ("0", "1"):
        monkeypatch.setenv("PULSE_GROUPED", flag)
        pol = PPOPolicy(device=DEV, seed=5)
        stats = pol.train_minibatch(obs, act, nlp, adv, ret, update_obs_rms=False, keep_grads=True).clone()
        torch.cuda.synchronize()
        results.append((stats, pol.flat.grads.clone(), pol.flat.params.clone()))
    torch.testing.assert_close(results[1][0], results[0][0], atol=1e-6, rtol=1e-6)
    torch.testing.assert_close(results[1][1], results[0][1], atol=1e-4, rtol=1e-3)
    torch.testing.assert_close(results[1][2], results[0][2], atol=1e-6, rtol=1e-5)
