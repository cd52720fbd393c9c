"""The update's links, element by element, against float64 references fed the kernels' own operands (tests/fp64_ref.py).

PPO with the AMP discriminator (one train_minibatch at the production minibatch, M = 16384 with B = 4096 AMP rows, and at a ragged
one, M = 5000 with B = 1000) in every GEMM mode -- default, PULSE_GEMM_BN=128, PULSE_GEMM_STAGES=4, PULSE_GROUPED=1 -- and the PULSE
VAE at the im_z_fit.yaml widths (optimize_kin(step=False) at M = 16384 and M = 4064).  Every link has its own tight bound, so a
missing k-block, a split-K slice added twice, a mask read from the wrong rows, a dropped bias column or a wrong coefficient fails
here even where the cosine checks of test_gpu_ppo.py / test_gpu_vae.py (against fp32 autograd) cannot see it.
Run with -s to print the margin of every link.
"""
import math

import pytest
import torch

from tests.fp64_ref import (U32, UBF, Gemm, Report, adam_ref, check, check_exact, check_mask, disc_loss_ref, f64, latent_loss_tol,
                            normalize_ref, ppo_loss_ref, silu64, silu_grad64, silu_grad_err, silu_tol, sum_tol, unpack_mask)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------------------------ shared pieces
def _snapshot(flat):
    torch.cuda.synchronize()
    return {"p": flat.params.clone(), "pb": flat.params_bf16.clone(), "m": flat.exp_avg.clone(), "v": flat.exp_avg_sq.clone(),
            "step": int(flat.step.item())}


def _w(snap, flat, l):
    """bf16 weight block [N, Kp] of layer l as the GEMMs read it (before Adam rewrote the mirror)."""
    off = flat.offset(l.w_idx)
    return snap["pb"][off:off + l.N * l.Kp].view(l.N, l.Kp)


def _b(snap, flat, l):
    """fp32 bias of a plain (not bias-augmented) layer as the forward epilogue read it."""
    off = flat.offset(l.b_idx)
    return snap["p"][off:off + l.N]


def _check_pads(rep, link, t, zero_from, one_col=None):
    if one_col is not None:
        check_exact(rep, link + " ones column", t[:, one_col], torch.ones_like(t[:, one_col]))
    if t.shape[1] > zero_from:
        check_exact(rep, link + " pads", t[:, zero_from:], torch.zeros_like(t[:, zero_from:]))


def check_mlp(rep, name, mlp, snap, x, dout, M):
    """Forward and backward links of one MLP from its training workspace.  Returns (dW per layer as Gemm, bias-gradient (ref, tol) per
    plain layer): the expected contributions of this backward pass to the flat gradients."""
    flat, ws, L = mlp.flat, mlp._ws[(M, True)], mlp.layers
    W = [_w(snap, flat, l) for l in L]
    bias = [None if mlp.aug else _b(snap, flat, l) for l in L]
    h = x
    for i, l in enumerate(L):
        g = Gemm(h[:M, :l.Kp], W[i].T, bias=bias[i])
        if i == len(L) - 1:
            g.check(rep, f"{name} L{i} head (fp32{', head1' if mlp._head1(i) else ''})", ws["out"][:M])
            break
        act = ws["act"][i]
        if l.act == "relu":
            check_mask(rep, f"{name} L{i} relu mask words", ws["mask"][i], g, l.N, M)
            check(rep, f"{name} L{i} act (relu, bf16)", act[:M, :l.N], torch.relu(g.y), g.tol(True), g.det_tol(True))
        elif l.act == "silu":
            g.check(rep, f"{name} L{i} pre (bf16)", ws["pre"][i][:M, :l.N])
            z = f64(ws["pre"][i][:M, :l.N])
            s = silu64(z)
            check(rep, f"{name} L{i} act (silu of the kernel's pre)", act[:M, :l.N], s, silu_tol(z, s))
        else:
            g.check(rep, f"{name} L{i} out (no activation, bf16)", act[:M, :l.N])
        _check_pads(rep, f"{name} L{i} act", act[:M], l.N + 1 if mlp.aug else l.N, l.N if mlp.aug else None)
        h = act
    wgrad, bgrad = {}, {}
    top, dy = len(L) - 1, dout
    if mlp._head1(top):
        head, hprev = L[top], ws["act"][top - 1][:M, :L[top].Kp]
        d = f64(dout[:M, 0])
        dh = (d[:, None] * f64(W[top][0])[None, :]) * (f64(hprev) > 0)            # products of two bf16: one rounding
        check_exact(rep, f"{name} head1 dh (gated, bf16)", ws["dact"][top - 1][:M, :head.Kp], dh.to(BF))
        wgrad[top] = Gemm(dout[:M, :1].T, hprev)
        if not mlp.aug:
            raise NotImplementedError("head1 bias gradients of plain layers are not exercised by these nets")
        dy, top = ws["dact"][top - 1], top - 1
    elif not mlp.aug:
        dd = f64(dout[:M, :L[top].N])
        bgrad[top] = (dd.sum(0), sum_tol(dd.abs().sum(0), M))                          # pulse_column_sum_bf16
    for i in reversed(range(top + 1)):
        l = L[i]
        x_in = x if i == 0 else ws["act"][i - 1]
        wgrad[i] = Gemm(dy[:M, :l.N].T, x_in[:M, :l.Kp])
        if i > 0:
            prev = L[i - 1]
            Wd = W[i][:, :prev.N] if mlp.aug else W[i]
            out = ws["dact"][i - 1][:M, :Wd.shape[1]]
            if prev.act == "relu":
                assert mlp.aug, "ReLU gates of plain layers are not exercised by these nets"
                g = Gemm(dy[:M, :l.N], Wd, gate=unpack_mask(ws["mask"][i - 1], prev.N, M))
                g.check(rep, f"{name} L{i} dgrad (mask-word gate)", out)
                y, acc = g.y, g.acc
            elif prev.act == "silu":
                g = Gemm(dy[:M, :l.N], Wd)
                z = f64(ws["pre"][i - 1][:M, :Wd.shape[1]])
                sg = silu_grad64(z)
                y = g.y * sg
                acc = g.acc * sg.abs() + g.y.abs() * silu_grad_err(z) + U32 * y.abs()
                check(rep, f"{name} L{i} dgrad (silu gate from the kernel's pre)", out, y, acc * (1 + UBF) + UBF * y.abs())
            else:
                g = Gemm(dy[:M, :l.N], Wd)
                g.check(rep, f"{name} L{i} dgrad (no gate)", out)
                y, acc = g.y, g.acc
            if not mlp.aug:                          # the dgrad epilogue's column sums are the bias gradient of the layer below
                bgrad[i - 1] = (y.sum(0)[:prev.N], (acc.sum(0) + sum_tol(y.abs().sum(0), M))[:prev.N])
            dy = ws["dact"][i - 1]
        elif mlp.input_grad_cols:
            Gemm(dy[:M, :l.N], W[0][:, :mlp.input_grad_cols]).check(rep, f"{name} dx (input columns, fp32)", ws["dx"][:M])
    return wgrad, bgrad


def check_grads(rep, name, mlp, wgrad, bgrad, extra=None):
    """flat.grads of every layer == this backward pass's contribution (+ `extra[i]` = (ref, tol) for terms added by other kernels)."""
    for i, l in enumerate(mlp.layers):
        g = wgrad[i]
        ref, tol, det = g.y, g.acc, g.det
        if extra is not None and i in extra:
            ref2, tol2 = extra[i]
            ref, tol, det = ref + ref2, tol + tol2 + 2 * U32 * (g.y.abs() + ref2.abs()), det + tol2 + 2 * U32 * (g.y.abs() + ref2.abs())
        check(rep, f"{name} L{i} dW total", l.weight_grad, ref, tol, det)
        if i in bgrad:
            check(rep, f"{name} L{i} db (column sums)", l.bias_grad, *bgrad[i])


def _merge64(mean, var, count, x):
    """RunningMeanStd training merge in float64 (batch mean / unbiased variance), and the fp32 mean / rstd the kernels then use."""
    x = f64(x)
    n = x.shape[0]
    bm, bv = x.mean(0), x.var(0, unbiased=True)
    tot = count + n
    delta = bm - mean
    var = (var * count + bv * n + delta * delta * count * n / tot) / tot
    mean = mean + delta * n / tot
    return mean, var, tot, mean.float(), 1.0 / torch.sqrt(var.float() + 1e-5)


def _check_normalized(rep, link, out, x, mean32, rstd32, cols, one_col, slack=0.0):
    y, tol = normalize_ref(x, mean32, rstd32)
    check(rep, link, out[:, :cols], y, tol + slack * y.abs())
    _check_pads(rep, link, out, one_col + 1 if one_col is not None else cols, one_col)


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


def _check_adam(rep, flat, snap, max_norm, lr, tag, expect_clip=None, grads=None):
    grads = flat.grads if grads is None else grads
    p1, m1, v1, dp, dm, dv, clipped, margin = adam_ref(snap["p"], grads, snap["m"], snap["v"], snap["step"], lr=lr, max_norm=max_norm)
    assert margin > 1e-4, f"{tag}: gradient norm within 1e-4 of max_norm: the clip decision is ambiguous"
    if expect_clip is not None:
        assert clipped == expect_clip, f"{tag}: clipping {'did not engage' if expect_clip else 'engaged'}"
    check(rep, f"adam {tag} params", flat.params, p1, dp)
    check(rep, f"adam {tag} exp_avg", flat.exp_avg, m1, dm)
    check(rep, f"adam {tag} exp_avg_sq", flat.exp_avg_sq, v1, dv)
    check_exact(rep, f"adam {tag} params_bf16 = bf16(params)", flat.params_bf16, flat.params.to(BF))
    assert int(flat.step.item()) == snap["step"] + 1, f"{tag}: step counter not advanced"
    assert float(flat.sumsq.item()) == 0.0, f"{tag}: gradient-norm accumulator not re-zeroed"
    return clipped


def _check_ppo_minibatch(rep, pol, M, B, snap, obs_stats, disc_stats, inputs):
    obs, actions, old_nlp, adv, ret, mus, amp = inputs
    b = pol._buf(M, True)
    x = b["x2"][0]
    _check_normalized(rep, "normalised obs (bf16)", x, obs, *obs_stats, 934, 934)
    dmu, dv = b["dmu"], b["dv"]
    # ---- actor and critic
    wa, ba = check_mlp(rep, "actor", pol.actor, snap, x, dmu, M)
    wc, bc = check_mlp(rep, "critic", pol.critic, snap, x, dv, M)
    mu, value = pol.actor._ws[(M, True)]["out"][:M], pol.critic._ws[(M, True)]["out"][:M]
    # ---- pulse_ppo_loss on the kernel's own mu / value
    ref = ppo_loss_ref(mu, value, actions, old_nlp, adv, ret, pol.logstd, old_mu=mus, e_clip=pol.e_clip, critic_coef=pol.critic_coef,
                       bounds_coef=pol.bounds_coef)
    amb = ref["ambiguous"]
    n_amb = int(amb.sum())
    assert n_amb <= max(2, 1e-3 * M), f"{n_amb} PPO rows lie within rounding of a branch threshold"
    r, adv64, mu64 = ref["ratio"], f64(adv), f64(mu)
    regimes = {"inside": int(((r > 0.8) & (r < 1.2)).sum()), "clipped above, adv > 0": int(((r > 1.2) & (adv64 > 0)).sum()),
               "clipped below, adv < 0": int(((r < 0.8) & (adv64 < 0)).sum()), "above, adv < 0 (unclipped)": int(((r > 1.2) & (adv64 < 0)).sum()),
               "|mu| > 1": int((mu64.abs() > 1).sum())}
    assert all(v > 0 for v in regimes.values()), regimes
    tol_mu = torch.where(amb[:, None], torch.full_like(ref["tol_mu"], math.inf), ref["tol_mu"])
    check(rep, "ppo_loss dmu (bf16)", dmu[:M, :69], ref["dmu"], tol_mu)
    rep.rows[-1] = rep.rows[-1][:3] + (f"{n_amb} of {M} rows",)
    _check_pads(rep, "ppo_loss dmu", dmu[:M], 69)
    check(rep, "ppo_loss dv (bf16)", dv[:M, 0], ref["dv"], ref["tol_v"])
    _check_pads(rep, "ppo_loss dv", dv[:M], 1)
    st = pol.stats.double()
    for k, name in enumerate(("sum a_loss", "sum c_loss", "sum b_loss", "sum kl", "clipped rows", "sum neglogp")):
        check(rep, f"ppo_loss stats[{k}] {name}", st[k:k + 1], ref["stats"][k].reshape(1), torch.as_tensor(ref["stats_tol"][k], dtype=torch.float64,
                                                                                                           device=DEV).reshape(1) + 1e-300)
    # ---- discriminator
    disc = pol.disc
    L1, L2, L3 = disc.mlp.layers
    db = disc._buf(B)
    xd = db["x"][0]
    mean, var, cnt = disc_stats
    for k, src in enumerate(amp):     # each batch is normalised with the statistics merged up to the batch before it
        m32, r32 = mean.float(), 1.0 / torch.sqrt(var.float() + 1e-5)
        _check_normalized(rep, f"disc normalised batch {k} (bf16)", xd[k * B:(k + 1) * B], src, m32, r32, 1960, 1960, slack=4 * U32)
        mean, var, cnt, _, _ = _merge64(mean, var, cnt, src)
    wd, bd = check_mlp(rep, "disc", disc.mlp, snap, xd, db["dlogit"], 3 * B)
    wsd = disc.mlp._ws[(3 * B, True)]
    gl, tl, dstats, dstats_tol = disc_loss_ref(wsd["out"][:3 * B], 2 * B, disc.disc_coef)
    check(rep, "disc_loss dlogit (bf16)", db["dlogit"][:3 * B, 0], gl, tl)
    _check_pads(rep, "disc_loss dlogit", db["dlogit"], 1)
    sd = disc.stats.double()
    for k in range(4):
        check(rep, f"disc_loss stats[{k}]", sd[k:k + 1], dstats[k].reshape(1).to(DEV),
              torch.as_tensor(dstats_tol[k], dtype=torch.float64, device=DEV).reshape(1) + 1e-300)
    # ---- gradient penalty chain on the demo rows (amp.py): masks are the demo rows' words, row stride 3B
    W1, W2 = _w(snap, pol.flat, L1), _w(snap, pol.flat, L2)
    w3 = snap["p"][pol.flat.offset(L3.w_idx):pol.flat.offset(L3.w_idx) + L3.Kp]
    m1 = unpack_mask(wsd["mask"][0][:, 2 * B:], L1.N, B)
    m2 = unpack_mask(wsd["mask"][1][:, 2 * B:], L2.N, B)
    h2 = f64(wsd["act"][1][2 * B:3 * B, :L2.N])
    check_exact(rep, "gp g2 = m2 * w3 (bf16)", db["g2"][:, :L2.N], torch.where(h2 > 0, f64(w3[:L2.N])[None, :], torch.zeros_like(h2)).to(BF))
    _check_pads(rep, "gp g2", db["g2"], L2.N)
    Gg1 = Gemm(db["g2"][:, :L2.N], W2[:, :L1.N], gate=m1)
    Gg1.check(rep, "gp g1 = m1 * (g2 W2) (bf16)", db["g1"][:, :L1.N])
    c = 2.0 * disc.disc_coef * disc.grad_penalty / B
    GG = Gemm(db["g1"][:, :L1.N], W1[:, :L1.K], alpha=c)
    GG.check(rep, "gp G = c * g1 W1 (bf16)", db["Gb"][:, :L1.K])
    _check_pads(rep, "gp G", db["Gb"], L1.K)
    sq_ref = (GG.y * GG.y).sum()
    sq_tol = (2 * GG.y.abs() * GG.acc + GG.acc ** 2).sum() + sum_tol((GG.y * GG.y).sum(), B * L1.K)
    check(rep, "gp stats[4] sum G^2", sd[4:5], sq_ref.reshape(1), sq_tol.reshape(1))
    pen1 = Gemm(db["g1"][:, :L1.N].T, db["Gb"])                                      # dW1 += g1^T G
    Gdu = Gemm(db["Gb"], W1.T, gate=m1)
    Gdu.check(rep, "gp du = m1 * (G W1^T) (bf16)", db["du"][:, :L1.N])
    pen2 = Gemm(db["g2"][:, :L2.N].T, db["du"][:, :L1.N])                          # dW2 += g2^T du
    Gs = Gemm(db["du"][:, :L1.N], W2[:, :L1.N].T, gate=m2)
    Gs.check(rep, "gp scratch = m2 * (du W2^T) (fp32)", db["scratch"][:, :L2.N])
    scr = f64(db["scratch"][:, :L2.N])
    pen3 = scr.sum(0)                                                               # dw3 += column sums, in fp32
    pen3_tol = sum_tol(scr.abs().sum(0), B)
    # ---- totals: prediction part + penalty part + 2 disc_coef (weight_decay [+ logit_reg]) w on the weight block
    p32 = lambda l: snap["p"][pol.flat.offset(l.w_idx):pol.flat.offset(l.w_idx) + l.N * l.Kp].view(l.N, l.Kp)
    extra = {}
    for i, l in enumerate((L1, L2, L3)):
        coef = 2.0 * disc.disc_coef * (disc.weight_decay + (disc.logit_reg if l is L3 else 0.0))
        reg = torch.zeros(l.N, l.Kp, dtype=torch.float64, device=DEV)
        reg[:, :l.K] = coef * f64(p32(l)[:, :l.K])
        y, t = reg.clone(), 2 * U32 * reg.abs()
        if l is L1:
            y, t = y + pen1.y, t + pen1.acc
        elif l is L2:
            y[:, :L1.N] += pen2.y
            t[:, :L1.N] += pen2.acc
        else:
            y[0, :L2.N] += pen3
            t[0, :L2.N] += pen3_tol
        extra[i] = (y, t + 2 * U32 * y.abs())
    check_grads(rep, "disc", disc.mlp, wd, bd, extra)
    wsq = [f64(p32(l)[:, :l.K]) ** 2 for l in (L1, L2, L3)]
    check(rep, "disc stats[5] sum w_logit^2", sd[5:6], wsq[2].sum().reshape(1), sum_tol(wsq[2].sum(), L3.K).reshape(1))
    check(rep, "disc stats[6] sum w^2", sd[6:7], sum(w.sum() for w in wsq).reshape(1),
          sum_tol(sum(w.sum() for w in wsq), sum(w.numel() for w in wsq)).reshape(1))
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


MODES = {"default": {}, "bn128": {"PULSE_GEMM_BN": "128"}, "stages4": {"PULSE_GEMM_STAGES": "4"}, "grouped": {"PULSE_GROUPED": "1"}}


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
