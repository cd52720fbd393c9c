"""PPO actor/critic path on the GPU vs the oracle / a plain PyTorch fp32 reference of the same ops.

Tolerances: the GEMMs run bf16 x bf16 -> fp32 (north_star: 'losses within 1e-3'); element-wise kernels are fp32.
"""
import ctypes as C
import math

import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _torch_mlp(mlp):
    """fp32 nn.Sequential with the same weights as a pulse_b200.nets.MLP."""
    mods = []
    for i, l in enumerate(mlp.layers):
        lin = torch.nn.Linear(l.K, l.N, device=DEV)
        with torch.no_grad():
            lin.weight.copy_(l.weight[:, :l.K])
            lin.bias.copy_(l.bias)
        mods.append(lin)
        if l.act == "relu":
            mods.append(torch.nn.ReLU())
        elif l.act == "silu":
            mods.append(torch.nn.SiLU())
    return torch.nn.Sequential(*mods)


def test_ppo_loss_kernel_matches_oracle():
    from oracle import pulse_oracle as po
    from pulse_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(0)
    M, A = 1000, 69
    mu = (torch.randn(M, A, device=DEV, generator=g) * 0.8).requires_grad_(True)
    value = torch.randn(M, 1, device=DEV, generator=g).requires_grad_(True)
    logstd = torch.full((A,), -2.9, device=DEV)
    actions = (mu.detach() + math.exp(-2.9) * torch.randn(M, A, device=DEV, generator=g)).contiguous()
    old_mu = (mu.detach() + 0.01 * torch.randn(M, A, device=DEV, generator=g)).contiguous()
    adv = torch.randn(M, device=DEV, generator=g)
    ret = torch.randn(M, device=DEV, generator=g)
    sigma = torch.exp(logstd).expand(M, A)
    old_nlp = po.gaussian_neglogp(actions, old_mu, sigma, logstd.expand(M, A)).contiguous()
    ref = po.ppo_total_loss(mu, value.squeeze(1), old_nlp, adv, ret, actions, logstd)
    ref["loss"].backward()
    dmu = torch.zeros(M, 72, device=DEV, dtype=torch.bfloat16)
    dmu_t = torch.zeros(72, M, device=DEV, dtype=torch.bfloat16)
    dv = torch.zeros(M, 8, device=DEV, dtype=torch.bfloat16)
    dv_t = torch.zeros(8, M, device=DEV, dtype=torch.bfloat16)
    stats = torch.zeros(6, device=DEV, dtype=torch.float64)
    mud, vd = mu.detach().contiguous(), value.detach().contiguous()
    a = _lib.PpoLossArgs(mu=mud.data_ptr(), ld_mu=A, value=vd.data_ptr(), ld_value=1, actions=actions.data_ptr(), old_neglogp=old_nlp.data_ptr(),
                         advantages=adv.data_ptr(), returns=ret.data_ptr(), old_mu=old_mu.data_ptr(), logstd=logstd.data_ptr(), num_actions=A,
                         e_clip=0.2, critic_coef=5.0, bounds_coef=10.0, dmu=dmu.data_ptr(), ld_dmu=72, dmu_t=dmu_t.data_ptr(), ld_dmu_t=M,
                         dvalue=dv.data_ptr(), ld_dv=8, dvalue_t=dv_t.data_ptr(), ld_dv_t=M, stats=stats.data_ptr())
    _lib.check(lib.pulse_ppo_loss(C.byref(a), M, _lib.current_stream()), "pulse_ppo_loss")
    torch.cuda.synchronize()
    s = stats.cpu() / M
    assert abs(s[0].item() - ref["a_loss"].item()) < 1e-4 * max(1, abs(ref["a_loss"].item()))  # exp(old - new) at fp32 round-off
    assert abs(s[1].item() - ref["c_loss"].item()) < 1e-4 * max(1, abs(ref["c_loss"].item()))
    assert abs(s[2].item() - ref["b_loss"].item()) < 1e-5
    assert abs(s[5].item() - ref["neglogp"].mean().item()) < 1e-3
    kl = po.policy_kl(mu.detach(), sigma, old_mu, sigma)
    assert abs(s[3].item() - kl.item()) < 1e-5
    torch.testing.assert_close(dmu[:, :A].float(), mu.grad, atol=2e-5, rtol=1e-2)
    torch.testing.assert_close(dmu_t[:A].float().T, mu.grad, atol=2e-5, rtol=1e-2)
    torch.testing.assert_close(dv[:, 0].float(), value.grad[:, 0], atol=2e-5, rtol=1e-2)
    torch.testing.assert_close(dv_t[0].float(), value.grad[:, 0], atol=2e-5, rtol=1e-2)


def test_normalize_and_moments_match_reference_semantics():
    from oracle import pulse_oracle as po
    from pulse_b200.ppo import RunningMeanStdB200
    g = torch.Generator(device=DEV).manual_seed(1)
    x1 = torch.randn(300, 934, device=DEV, generator=g) * 3 + 1
    x2 = torch.randn(5000, 934, device=DEV, generator=g) * 0.5 - 2
    rms = RunningMeanStdB200(934, DEV)
    ref = po.RunningMeanStd(934)
    out = torch.zeros(300, 960, device=DEV, dtype=torch.bfloat16)
    out_t = torch.zeros(960, 300, device=DEV, dtype=torch.bfloat16)
    for x in (x1, x2):
        rms.update(x)
        ref.update(x.cpu())
    # the reference takes the batch mean / var in fp32 (input.mean / input.var) before the fp64 merge; the kernel
    # accumulates the batch sums in fp64, so agreement is at fp32 round-off, not fp64
    torch.testing.assert_close(rms.running_mean.cpu(), ref.mean, atol=2e-6, rtol=2e-6)
    torch.testing.assert_close(rms.running_var.cpu(), ref.var, atol=2e-5, rtol=2e-5)
    rms.normalize_into(x1, out, out_t)
    y = ref.normalize(x1.cpu())
    torch.testing.assert_close(out[:, :934].float().cpu(), y, atol=2e-2, rtol=1e-2)   # bf16 rounding of values in [-5, 5]
    assert torch.all(out[:, 934:] == 0)
    assert torch.equal(out_t.T.contiguous(), out)


@pytest.mark.parametrize("rows,cols", [(300, 934), (4096, 1960), (37, 10), (64, 7)])
def test_fused_normalize_moments_equals_two_pass(rows, cols):
    """pulse_normalize_moments (one pass) == normalise with the OLD statistics, then merge (running_mean_std.py:91-107)."""
    from oracle import pulse_oracle as po
    from pulse_b200.nets import pad8
    from pulse_b200.ppo import RunningMeanStdB200
    g = torch.Generator(device=DEV).manual_seed(rows + cols)
    fused, two, ref = RunningMeanStdB200(cols, DEV), RunningMeanStdB200(cols, DEV), po.RunningMeanStd(cols)
    for k in range(3):
        x = torch.randn(rows, cols, device=DEV, generator=g) * (k + 1) + k
        o1 = torch.full((rows, pad8(cols)), 7.0, device=DEV, dtype=torch.bfloat16)
        o2 = torch.zeros_like(o1)
        fused.normalize_update(x, o1)
        two.normalize_into(x, o2)
        two.update(x)
        y = ref.normalize(x.cpu())
        ref.update(x.cpu())
        assert torch.equal(o1, o2)                       # same fp32 arithmetic, same bf16 rounding, padding zeroed
        torch.testing.assert_close(o1[:, :cols].float().cpu(), y, atol=2e-2, rtol=1e-2)
        torch.testing.assert_close(fused.running_mean, two.running_mean, atol=1e-12, rtol=1e-12)
        torch.testing.assert_close(fused.running_var, two.running_var, atol=1e-10, rtol=1e-10)
        torch.testing.assert_close(fused.running_mean.cpu(), ref.mean, atol=5e-6, rtol=5e-6)
        assert float(fused.count) == float(two.count) == 1 + (k + 1) * rows
    assert torch.all(fused._sums == 0)


def test_policy_forward_and_update_match_fp32_reference():
    from oracle import pulse_oracle as po
    from pulse_b200.ppo import PPOPolicy
    pol = PPOPolicy(device=DEV, seed=3)
    actor_ref, critic_ref = _torch_mlp(pol.actor), _torch_mlp(pol.critic)
    g = torch.Generator(device=DEV).manual_seed(4)
    M = 2048
    obs = torch.randn(M, 934, device=DEV, generator=g) * 2
    pol.obs_rms.update(obs)
    pol.obs_rms.frozen = True
    eps = torch.randn(M, 69, device=DEV, generator=g)
    out = pol.act(obs, eps=eps)
    xn = torch.clamp((obs - pol.obs_rms.mean_f32) * pol.obs_rms.rstd_f32, -5, 5)
    mu_ref, v_ref = actor_ref(xn), critic_ref(xn)
    torch.testing.assert_close(out["mus"], mu_ref, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(out["values"], v_ref, atol=2e-2, rtol=2e-2)  # value_rms is identity at init (mean 0, var 1)
    sigma = torch.exp(pol.logstd).expand(M, 69)
    torch.testing.assert_close(out["actions"], out["mus"] + sigma * eps, atol=1e-6, rtol=1e-6)
    nlp = po.gaussian_neglogp(out["actions"], out["mus"], sigma, pol.logstd.expand(M, 69))
    torch.testing.assert_close(out["neglogpacs"], nlp, atol=1e-3, rtol=1e-5)

    # one PPO minibatch: losses within 1e-3, gradients aligned with fp32 autograd, Adam step applied
    actions, old_nlp = out["actions"].clone(), out["neglogpacs"].clone()
    adv = torch.randn(M, device=DEV, generator=g)
    ret = torch.randn(M, device=DEV, generator=g)
    w_before = pol.flat.params.clone()
    ref = po.ppo_total_loss(mu_ref, v_ref.squeeze(1), old_nlp, adv, ret, actions, pol.logstd)
    ref["loss"].backward()
    stats = pol.train_minibatch(obs, actions, old_nlp, adv, ret, old_mu=out["mus"].clone(), update_obs_rms=False, keep_grads=True).cpu() / M
    torch.cuda.synchronize()
    for k, i in (("a_loss", 0), ("c_loss", 1), ("b_loss", 2)):
        assert abs(stats[i].item() - ref[k].item()) < 1e-3 * max(1.0, abs(ref[k].item())), (k, stats[i].item(), ref[k].item())
    for mlp, refm in ((pol.actor, actor_ref), (pol.critic, critic_ref)):
        lins = [m for m in refm if isinstance(m, torch.nn.Linear)]
        for l, lin in zip(mlp.layers, lins):
            gw, gb = l.weight_grad[:, :l.K], l.bias_grad
            cos = torch.nn.functional.cosine_similarity(gw.flatten(), lin.weight.grad.flatten(), dim=0)
            assert cos > 0.995, (l.N, l.K, cos.item())
            rel = (gw - lin.weight.grad).norm() / lin.weight.grad.norm()
            assert rel < 0.15, rel.item()  # bf16 activations / gradients, ReLU masks that flip near zero
            cosb = torch.nn.functional.cosine_similarity(gb, lin.bias.grad, dim=0)
            assert cosb > 0.995, cosb.item()
            assert torch.all(l.weight_grad[:, l.pad_start:] == 0)     # zero padding never receives a gradient (column K is the bias)
    # Adam: compare against torch.optim.Adam fed the SAME (our) gradients
    p = w_before.clone().requires_grad_(True)
    p.grad = pol.flat.grads.clone()
    torch.nn.utils.clip_grad_norm_([p], 50.0)
    opt = torch.optim.Adam([p], lr=2e-5, eps=1e-8)
    opt.step()
    torch.testing.assert_close(pol.flat.params, p.detach(), atol=1e-7, rtol=1e-5)
    l0 = pol.actor.layers[0]
    torch.testing.assert_close(l0.w_bf16.float(), l0.weight, atol=1e-2, rtol=1e-2)
    # checkpoint keys follow the rl_games layout the reference's loaders read (network_loader.py:81-99)
    sd = pol.state_dict()
    for k in ("a2c_network.actor_mlp.0.weight", "a2c_network.actor_mlp.2.bias", "a2c_network.mu.weight", "a2c_network.critic_mlp.0.weight",
              "a2c_network.value.bias", "a2c_network.sigma", "running_mean_std.running_mean"):
        assert k in sd
    assert sd["a2c_network.actor_mlp.0.weight"].shape == (1024, 934) and sd["a2c_network.mu.weight"].shape == (69, 512)


def test_disc_loss_and_gradient_penalty_match_autograd():
    """AMP discriminator: analytic gradient penalty (GEMM chain) vs the oracle's autograd double backward, im.yaml sizes."""
    from oracle import pulse_oracle as po
    from pulse_b200.ppo import PPOPolicy
    pol = PPOPolicy(device=DEV, seed=7, with_disc=True)
    disc = pol.disc
    B = 4096                                   # amp_minibatch_size (im.yaml:81)
    g = torch.Generator(device=DEV).manual_seed(8)
    agent, replay, demo = (torch.randn(B, 1960, device=DEV, generator=g) for _ in range(3))
    demo = demo * 0.7 + 0.3
    ref_mlp = _torch_mlp(disc.mlp)
    lins = [m for m in ref_mlp if isinstance(m, torch.nn.Linear)]
    xn = lambda x: torch.clamp((x - disc.rms.mean_f32) * disc.rms.rstd_f32, -5, 5)
    ref = po.disc_loss(ref_mlp, xn(agent), xn(replay), xn(demo), lins[-1].weight, [l.weight for l in lins])
    (ref["disc_loss"] * 5.0).backward()
    pol.flat.zero_grad()
    stats = disc.loss_backward(agent, replay, demo, update_rms=False)
    torch.cuda.synchronize()
    out = disc.loss_from_stats(stats, B)
    # north_star: losses within 1e-3 (relative), every term
    assert abs(out["disc_loss"] - ref["disc_loss"].item()) < 1e-3 * abs(ref["disc_loss"].item()), (out, ref["disc_loss"].item())
    assert abs(out["disc_grad_penalty"] - ref["disc_grad_penalty"].item()) < 1e-3 * ref["disc_grad_penalty"].item(), (out, ref["disc_grad_penalty"].item())
    assert abs(out["disc_logit_loss"] - ref["disc_logit_loss"].item()) < 1e-3 * ref["disc_logit_loss"].item()
    assert abs(out["disc_agent_acc"] - ref["disc_agent_acc"].item()) < 0.02 and abs(out["disc_demo_acc"] - ref["disc_demo_acc"].item()) < 0.02
    for l, lin in zip(disc.mlp.layers, lins):
        gw = l.weight_grad[:, :l.K]
        cos = torch.nn.functional.cosine_similarity(gw.flatten(), lin.weight.grad.flatten(), dim=0)
        rel = (gw - lin.weight.grad).norm() / lin.weight.grad.norm()
        assert cos > 0.99 and rel < 0.15, (l.N, l.K, cos.item(), rel.item())
        cosb = torch.nn.functional.cosine_similarity(l.bias_grad, lin.bias.grad, dim=0)
        assert cosb > 0.99, (l.N, cosb.item())
    # rewards: -log(max(1 - sigmoid(D), 1e-4)) * 2
    r = disc.rewards(agent)
    torch.testing.assert_close(r, po.disc_reward(ref_mlp(xn(agent)).detach()), atol=3e-2, rtol=3e-2)


@pytest.mark.parametrize("rows,k", [(1000, 512), (37, 64), (4096, 2048), (5, 8)])
def test_single_output_head_kernels(rows, k):
    """pulse_head1_forward / pulse_head1_backward against fp32 torch on the same bf16 operands."""
    from pulse_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(rows * 7 + k)
    h = torch.relu(torch.randn(rows, k, device=DEV, generator=g)).bfloat16()
    w = (torch.randn(k, device=DEV, generator=g) * 0.1).bfloat16()
    bias = torch.randn(1, device=DEV, generator=g)
    dv = torch.zeros(rows, 8, device=DEV, dtype=torch.bfloat16)
    dv[:, 0] = (torch.randn(rows, device=DEV, generator=g) * 0.01).bfloat16()
    out = torch.zeros(rows, 1, device=DEV)
    st = _lib.current_stream(DEV)
    _lib.check(lib.pulse_head1_forward(h.data_ptr(), h.stride(0), rows, k, w.data_ptr(), bias.data_ptr(), out.data_ptr(), 1, st), "fwd")
    ref = h.float() @ w.float() + bias
    torch.testing.assert_close(out[:, 0], ref, atol=1e-4, rtol=1e-4)
    dh = torch.full((rows, k), 3.0, device=DEV, dtype=torch.bfloat16)
    dw, db, dbp = torch.ones(k, device=DEV), torch.ones(1, device=DEV), torch.ones(k, device=DEV)
    part = torch.empty(_lib.HEAD1_MAX_CTAS * (2 * k + 1), device=DEV)
    _lib.check(lib.pulse_head1_backward(h.data_ptr(), h.stride(0), rows, k, dv.data_ptr(), dv.stride(0), w.data_ptr(), dh.data_ptr(), dh.stride(0),
                                        dw.data_ptr(), db.data_ptr(), dbp.data_ptr(), part.data_ptr(), st), "bwd")
    d = dv[:, 0].float()
    dh_ref = d[:, None] * w.float()[None, :] * (h.float() > 0)
    assert torch.equal(dh, dh_ref.bfloat16())                          # single products: exact up to the bf16 rounding
    torch.testing.assert_close(dw, 1 + (d[:, None] * h.float()).sum(0), atol=1e-4, rtol=1e-4)   # ADDS into the gradient buffers
    torch.testing.assert_close(db, 1 + d.sum().reshape(1), atol=1e-5, rtol=1e-4)
    torch.testing.assert_close(dbp, 1 + dh_ref.sum(0), atol=1e-4, rtol=1e-4)


def test_prefetched_minibatch_sequence_equals_inline_sequence():
    """train_minibatch(prepared=True, prefetch=next) -- the next minibatch's normalisation + running-statistics updates prepared
    on a side stream into the other operand slot -- must leave the same weights, normalisers and loss statistics as the inline
    sequence (same order of statistics updates as calc_gradients: batch i, then batch i+1)."""
    from pulse_b200.ppo import PPOPolicy
    g = torch.Generator(device=DEV).manual_seed(11)
    M, B, n = 1024, 512, 4
    obs = [torch.randn(M, 934, device=DEV, generator=g) * (1 + k) for k in range(n)]
    eps = [torch.randn(M, 69, device=DEV, generator=g) for _ in range(n)]
    adv = [torch.randn(M, device=DEV, generator=g) for _ in range(n)]
    ret = [torch.randn(M, device=DEV, generator=g) for _ in range(n)]
    amp = [tuple(torch.randn(B, 1960, device=DEV, generator=g) * (1 + 0.5 * k) for _ in range(3)) for k in range(n)]
    results = []
    for mode in ("inline", "start", "loss", "reduce"):
        pol = PPOPolicy(device=DEV, seed=5, with_disc=True)
        act, mu, nlp = [], [], []
        for i in range(n):                           # rollout-consistent actions / neglogp / mus (probability ratios near 1)
            out = pol.act(obs[i], eps=eps[i])
            act.append(out["actions"].clone()), mu.append(out["mus"].clone()), nlp.append(out["neglogpacs"].clone())
        if mode != "inline":
            os.environ["PULSE_PREFETCH_AT"] = mode
            pol.prepare_inputs(obs[0], amp[0], slot=0)
        try:
            for rep in range(2):                     # two passes over the minibatches, like two mini-epochs
                for i in range(n):
                    kw = {}
                    if mode != "inline":
                        last = rep == 1 and i == n - 1
                        kw = dict(slot=i & 1, prepared=True, prefetch=None if last else (obs[(i + 1) % n], amp[(i + 1) % n]))
                    pol.train_minibatch(obs[i], act[i], nlp[i], adv[i], ret[i], old_mu=mu[i], amp=amp[i], **kw)
        finally:
            os.environ.pop("PULSE_PREFETCH_AT", None)
        torch.cuda.synchronize()
        results.append((pol.flat.params.clone(), pol.obs_rms.running_mean.clone(), pol.obs_rms.count.clone(),
                        pol.disc.rms.running_var.clone(), pol.stats.clone(), pol.disc.stats.clone()))
    base = results[0]
    for mode, res in zip(("start", "loss", "reduce"), results[1:]):
        for k, (a, b) in enumerate(zip(base, res)):
            if k == 0:               # weights: the fp32 reductions of the weight gradients are order-dependent in the last bits, and
                d = (a - b).abs()    # Adam turns a sign flip of a ~0 gradient into 2 * lr; 8 steps at lr 2e-5 bound the worst case
                assert d.mean().item() < 1e-6 and d.max().item() < 5e-4, (mode, d.mean().item(), d.max().item())
            elif k in (4, 5):        # loss sums
                torch.testing.assert_close(a, b, atol=1e-6, rtol=2e-4, msg=lambda m: f"{mode} item {k}: {m}")
            else:                    # running statistics: the same kernels on the same data in the same order.  The fp64 atomics add in a
                # run-dependent order (last bits of sums of O(1) values: ~1e-16 absolute), so an element that happens to lie near zero has
                # no meaningful RELATIVE error: the absolute floor covers it (seen once in ~8 full-suite runs with atol = 0)
                torch.testing.assert_close(a, b, atol=1e-12, rtol=1e-11, msg=lambda m: f"{mode} item {k}: {m}")
