"""The update's links, element by element, against float64 references fed the kernels' own operands (tests/fp64_ref.py).

PPO with the AMP discriminator (one train_minibatch at the production minibatch, M = 16384 with B = 4096 AMP rows, and at a ragged
one, M = 5000 with B = 1000) in every GEMM mode -- default, PULSE_GEMM_BN=128, PULSE_GEMM_STAGES=4 -- and the PULSE
VAE at the im_z_fit.yaml widths (optimize_kin(step=False) at M = 16384 and M = 4064).  Every link has its own tight bound, so a
missing k-block, a split-K slice added twice, a mask read from the wrong rows, a dropped bias column or a wrong coefficient fails
here even where the cosine checks of test_gpu_ppo.py / test_gpu_vae.py (against fp32 autograd) cannot see it.
Run with -s to print the margin of every link.
"""
import pytest
import torch

from tests.fp64_links import (_check_adam, _check_normalized, _check_pads, _snapshot, check_disc, check_grads, check_mlp,
                               check_ppo_loss)
from tests.fp64_ref import U32, UBF, Report, check, check_exact, f64, latent_loss_tol

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------------------------------ PPO + AMP
def _ppo_inputs(pol, M, B, g):
    """One minibatch whose rows cover every branch of the PPO loss: ratio inside the clip range, clipped above with adv > 0, clipped
    below with adv < 0, and above the range with adv < 0 (unclipped, gradient flows).  old_neglogp is perturbed per row group."""
    obs = torch.randn(M, 934, device=DEV, generator=g) * 1.5 + 0.2
    eps = torch.randn(M, 69, device=DEV, generator=g)
    out = pol.act(obs, eps=eps)
    actions, nlp, mus = out["actions"].clone(), out["neglogpacs"].clone(), out["mus"].clone()
    adv = torch.randn(M, device=DEV, generator=g)
    grp = torch.arange(M, device=DEV) % 4
    nlp = nlp + torch.where(grp == 1, 0.4, torch.where(grp == 2, -0.4, torch.where(grp == 3, 0.4, 0.0)))
    adv = torch.where(grp == 1, adv.abs() + 0.1, torch.where(grp >= 2, -(adv.abs() + 0.1), adv))
    ret = torch.randn(M, device=DEV, generator=g)
    amp = tuple(torch.randn(B, 1960, device=DEV, generator=g) * s + o for s, o in ((1.0, 0.0), (1.3, 0.2), (0.7, 0.3)))
    return obs, actions, nlp, adv, ret, mus, amp


def _check_ppo_minibatch(rep, pol, M, B, snap, obs_stats, disc_stats, inputs):
    obs, actions, old_nlp, adv, ret, mus, amp = inputs
    x = pol._buf(M, True)["x2"][0]
    _check_normalized(rep, "normalised obs (bf16)", x, obs, *obs_stats, pol.obs_size, pol.obs_size)
    wa, ba = check_mlp(rep, "actor", pol.actor, snap, x, pol._buf(M, True)["dmu"], M)
    wc, bc = check_mlp(rep, "critic", pol.critic, snap, x, pol._buf(M, True)["dv"], M)
    check_ppo_loss(rep, pol, M, actions, old_nlp, adv, ret, mus)
    check_disc(rep, pol, B, snap, disc_stats, amp)
    check_grads(rep, "actor", pol.actor, wa, ba)
    check_grads(rep, "critic", pol.critic, wc, bc)


def _new_policy(seed):
    from pulse_b200.ppo import PPOPolicy
    pol = PPOPolicy(device=DEV, seed=seed, with_disc=True)
    head = pol.actor.layers[-1]
    with torch.no_grad():             # bias a few action heads past the soft bound so the bounds loss has active elements
        head.weight[:4, head.K] = torch.tensor([1.5, -1.5, 1.2, -1.2], device=DEV)
        head.refresh()
    g = torch.Generator(device=DEV).manual_seed(seed + 100)
    pol.obs_rms.update(torch.randn(4096, 934, device=DEV, generator=g) * 1.3 + 0.1)      # non-trivial normalisers
    pol.disc.rms.update(torch.randn(4096, 1960, device=DEV, generator=g) * 0.9 - 0.1)
    return pol, g


def _disc_stats(pol):
    r = pol.disc.rms
    return f64(r.running_mean).clone(), f64(r.running_var).clone(), float(r.count)


MODES = {"default": {}, "bn128": {"PULSE_GEMM_BN": "128"}, "stages4": {"PULSE_GEMM_STAGES": "4"}}


@pytest.mark.parametrize("M,B", [(16384, 4096), (5000, 1000)])
@pytest.mark.parametrize("mode", list(MODES))
def test_ppo_amp_update_links_fp64(monkeypatch, mode, M, B):
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    pol, g = _new_policy(seed=M + B)
    rep = Report(f"PPO + AMP update, M={M}, B={B}, mode={mode}")
    steps = 1 if M == 16384 else 3     # the ragged case also runs Adam over three consecutive minibatches
    norm1 = None
    try:
        for step in range(steps):
            inputs = _ppo_inputs(pol, M, B, g)
            snap = _snapshot(pol.flat)
            obs_stats = (pol.obs_rms.mean_f32.clone(), pol.obs_rms.rstd_f32.clone())
            disc_stats = _disc_stats(pol)
            if steps > 1:      # clipping off, on, off: max_norm far above, then far below the norm of the first step's gradients
                pol.grad_norm = 0.25 * norm1 if step == 1 else 1e9
            pol.reset_stats()
            obs, actions, old_nlp, adv, ret, mus, amp = inputs
            pol.train_minibatch(obs, actions, old_nlp, adv, ret, old_mu=mus, amp=amp, keep_grads=True)
            torch.cuda.synchronize()
            if step == 0:
                _check_ppo_minibatch(rep, pol, M, B, snap, obs_stats, disc_stats, inputs)
                norm1 = float(f64(pol.flat.grads).norm())
            _check_adam(rep, pol.flat, snap, pol.grad_norm, pol.lr, f"step {step + 1}", expect_clip=(step == 1) if steps > 1 else None)
        if steps > 1:          # one more optimizer step on the kept gradients, this time clearing them
            snap = _snapshot(pol.flat)
            grads = pol.flat.grads.clone()
            pol.flat.adam_step(pol.lr, max_norm=50.0, zero_grads=True)
            torch.cuda.synchronize()
            _check_adam(rep, pol.flat, snap, 50.0, pol.lr, "step 4 (zero_grads)", grads=grads)
            assert float(pol.flat.grads.abs().max()) == 0.0, "zero_grads=True left gradients behind"
    finally:
        print("\n" + rep.text())


# ------------------------------------------------------------------------------------------------------------------------------ VAE
@pytest.mark.parametrize("M", [16384, 4064])
def test_vae_optimize_kin_links_fp64(M):
    from oracle import pulse_oracle as po
    from pulse_b200.vae import PulseVAE
    vae = PulseVAE(device=DEV, seed=2, with_critic=False)
    E, S, A, T = vae.E, vae.S, vae.A, vae.horizon
    g = torch.Generator(device=DEV).manual_seed(M)
    vae.obs_rms.update(torch.randn(4096, vae.obs_size, device=DEV, generator=g) * 1.2 + 0.1)
    obs = torch.randn(M, vae.obs_size, device=DEV, generator=g) * 1.5
    gt = torch.randn(M, A, device=DEV, generator=g) * 0.3
    noise = torch.randn(M, E, device=DEV, generator=g)
    NE = M // T
    prog = (torch.arange(T, device=DEV)[None, :] + torch.randint(0, 50, (NE, 1), device=DEV, generator=g)).clone()
    prog[::5, 7:] = torch.arange(T - 7, device=DEV)[None, :]          # resets inside the horizon: pairs the AR(1) term must skip
    prog = prog.reshape(M)
    snap = _snapshot(vae.flat)
    m32, r32 = vae.obs_rms.mean_f32.clone(), vae.obs_rms.rstd_f32.clone()
    rep = Report(f"VAE optimize_kin, M={M}")
    try:
        vae.optimize_kin(obs, gt, prog, noise=noise, step=False)
        torch.cuda.synchronize()
        b = vae._buf(M)
        x = b["x"]
        _check_normalized(rep, "normalised obs (bf16)", x, obs, m32, r32, vae.obs_size, None)
        check_exact(rep, "copy_cols prior_in", b["prior_in"][:, :S], x[:, :S])
        _check_pads(rep, "copy_cols prior_in", b["prior_in"], S)
        check_exact(rep, "copy_cols dec_in self window", b["dec_in"][:, E:E + S], x[:, :S])
        _check_pads(rep, "copy_cols dec_in", b["dec_in"], E + S)
        we, be = check_mlp(rep, "enc", vae.enc, snap, x, b["d_enc"], M)
        head = vae.enc._ws[(M, True)]["out"][:M]
        qm, lv = f64(head[:, :E]), torch.clamp(f64(head[:, E:]), vae.clamp_lo, vae.clamp_hi)
        en = torch.exp(0.5 * lv) * f64(noise)
        z = qm + en
        check(rep, "reparam z -> dec_in[:, :E] (bf16)", b["dec_in"][:, :E], z, UBF * z.abs() + 6 * U32 * (qm.abs() + en.abs() * (1 + lv.abs())))
        pred = vae.dec._ws[(M, True)]["out"][:M]
        d = f64(pred) - f64(gt)
        nrm = d.norm(dim=-1, keepdim=True)
        gp = torch.where(nrm > 0, d / (nrm * M), torch.zeros_like(d))
        check(rep, "action loss dpred (bf16)", b["dpred"][:, :A], gp, (UBF + 16 * U32) * gp.abs() * (1 + UBF))
        _check_pads(rep, "action loss dpred", b["dpred"], A)
        wdec, bdec = check_mlp(rep, "dec", vae.dec, snap, b["dec_in"], b["dpred"], M)
        wp, bp = check_mlp(rep, "prior", vae.prior, snap, b["prior_in"], b["d_prior"], M)
        # ---- latent losses: float64 autograd of the oracle's expressions on the kernel's heads, noise, dz and progress
        prior_head = vae.prior._ws[(M, True)]["out"][:M]
        dz = vae.dec._ws[(M, True)]["dx"][:M]
        e, p = f64(head).requires_grad_(True), f64(prior_head).requires_grad_(True)
        qm_, qv_ = e[:, :E], torch.clamp(e[:, E:], vae.clamp_lo, vae.clamp_hi)
        pm_, pv_ = p[:, :E], torch.clamp(p[:, E:], vae.clamp_lo, vae.clamp_hi)
        kld = po.kl_multi(qm_, qv_, pm_, pv_).mean()
        tz = qm_.view(NE, T, E)
        err = tz[:, 1:] - tz[:, :-1] * 0.99
        idx = prog.view(NE, T, 1)
        keep = ~(((idx[:, 1:] - idx[:, :-1]) != 1) | (idx <= 2)[:, 1:] | (idx <= 2)[:, :-1])
        ar1 = torch.norm((err * keep.double()).reshape(-1, E), dim=-1).mean()
        zz = qm_ + torch.exp(0.5 * qv_) * f64(noise)
        loss = vae.kld_coefficient * kld + vae.ar1_coefficient * ar1 + (zz * f64(dz)).sum()
        ge, gpr = torch.autograd.grad(loss, (e, p))
        te, tp = latent_loss_tol(head, prior_head, noise, dz, prog, E, T, vae.kld_coefficient, vae.ar1_coefficient)
        check(rep, "latent loss d_enc (bf16)", b["d_enc"], ge, UBF * ge.abs() + te * (1 + UBF))
        check(rep, "latent loss d_prior (bf16)", b["d_prior"], gpr, UBF * gpr.abs() + tp * (1 + UBF))
        check_grads(rep, "enc", vae.enc, we, be)
        check_grads(rep, "prior", vae.prior, wp, bp)
        check_grads(rep, "dec", vae.dec, wdec, bdec)
    finally:
        print("\n" + rep.text())
