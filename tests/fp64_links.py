"""Link checkers of the update shared by tests/test_gpu_update_fp64.py and tests/test_gpu_sept_fp64.py: each reads the operands a net's
kernels stored in its workspaces and holds every GEMM / element-wise link to its own bound from tests/fp64_ref.py.  Plain torch: they
run on the CPU as well (tests/test_sept_fp64_cpu.py feeds them simulated kernels)."""
import math

import torch

from tests.fp64_ref import (U32, U64, UBF, Gemm, adam_ref, check, check_exact, check_mask, disc_loss_ref, f64, normalize_ref, ppo_loss_ref,
                            silu64, silu_gated, silu_gemm_tol, silu_tol, sum_tol, unpack_mask)

BF = torch.bfloat16


def _sync(t):
    if t.is_cuda:
        torch.cuda.synchronize(t.device)


def _snapshot(flat):
    _sync(flat.params)
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


def check_mlp(rep, name, mlp, snap, x, dout, M, top_out=None):
    """Forward and backward links of one MLP from its training workspace.  Returns (dW per layer as Gemm, bias-gradient (ref, tol) per
    plain layer): the expected contributions of this backward pass to the flat gradients.
    Headless nets (mlp.headless): the top layer's SiLU activation is read from `top_out` (the window forward(out=) wrote it into; its
    workspace buffer otherwise) and `dout` is the gradient w.r.t. the top PRE-activation, already gated by the caller."""
    flat, ws, L = mlp.flat, mlp._ws[(M, True)], mlp.layers
    W = [_w(snap, flat, l) for l in L]
    bias = [None if mlp.aug else _b(snap, flat, l) for l in L]
    h = x
    for i, l in enumerate(L):
        g = Gemm(h[:M, :l.Kp], W[i].T, bias=bias[i])
        if i == len(L) - 1 and not mlp.headless:
            g.check(rep, f"{name} L{i} head (fp32{', head1' if mlp._head1(i) else ''})", ws["out"][:M])
            break
        act = ws["act"][i]
        window = i == len(L) - 1 and top_out is not None
        if window:
            act = top_out
        if l.act == "relu":
            check_mask(rep, f"{name} L{i} relu mask words", ws["mask"][i], g, l.N, M)
            check(rep, f"{name} L{i} act (relu, bf16)", act[:M, :l.N], torch.relu(g.y), g.tol(True), g.det_tol(True))
        elif l.act == "silu":
            g.check(rep, f"{name} L{i} pre (bf16)", ws["pre"][i][:M, :l.N])
            z = f64(ws["pre"][i][:M, :l.N])
            s = silu64(z)
            check(rep, f"{name} L{i} act (silu of the kernel's pre{', in the window' if window else ''})", act[:M, :l.N], s, silu_tol(z, s))
        else:
            g.check(rep, f"{name} L{i} out (no activation, bf16)", act[:M, :l.N])
        if not window:               # past a caller's window lie the caller's columns, not pads
            _check_pads(rep, f"{name} L{i} act", act[:M], l.N + 1 if mlp.aug else l.N, l.N if mlp.aug else None)
        h = act
    wgrad, bgrad = {}, {}
    top, dy = len(L) - 1, dout
    if mlp.headless:
        pass
    elif mlp._head1(top):
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
                y, acc = silu_gated(Gemm(dy[:M, :l.N], Wd), ws["pre"][i - 1][:M, :Wd.shape[1]])
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


def check_mlp_eval(rep, name, mlp, snap, x, M, top_out=None, slot=0):
    """Forward links of one MLP from its evaluation workspace `slot` (no pre-activation stored: a SiLU is applied to the fp32 accumulator,
    fp64_ref.silu_gemm_tol).  The top output is read from `top_out` when given: the activation window of a headless net, or the fp32
    head a headed net wrote through forward(out=) (an experience slice, any row stride).  A head1 top layer (pulse_head1_forward, the
    GEMV of a single-output head on a ReLU layer) is a Gemm over its bf16 input and weight row -- with a bias-augmented net the input's
    ones column times the bias column, otherwise one fp32 bias add."""
    ws, L = mlp._ws[(M, False) if slot == 0 else (M, False, slot)], mlp.layers
    h = x
    for i, l in enumerate(L):
        g = Gemm(h[:M, :l.Kp], _w(snap, mlp.flat, l).T, bias=None if mlp.aug else _b(snap, mlp.flat, l))
        if i == len(L) - 1 and not mlp.headless:
            out = ws["out"] if top_out is None else top_out
            where = ", in the slice" if top_out is not None else ""
            g.check(rep, f"{name} L{i} eval head (fp32{', head1 GEMV' if mlp._head1(i) else ''}{where})", out[:M, :l.N])
            break
        window = i == len(L) - 1 and top_out is not None
        act = top_out if window else ws["act"][i]
        if l.act == "silu":
            check(rep, f"{name} L{i} eval act (silu of the fp32 accumulator{', in the window' if window else ''})", act[:M, :l.N],
                  silu64(g.y), silu_gemm_tol(g))
        elif l.act == "relu":
            check(rep, f"{name} L{i} eval act (relu, bf16)", act[:M, :l.N], torch.relu(g.y), g.tol(True), g.det_tol(True))
        else:
            g.check(rep, f"{name} L{i} eval out (no activation, bf16)", act[:M, :l.N])
        if not window:
            _check_pads(rep, f"{name} L{i} eval act", act[:M], l.N + 1 if mlp.aug else l.N, l.N if mlp.aug else None)
        h = act


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


def _merge64_tol(mean, var, count, x):
    """Bound of |kernel - _merge64| for one merge (pulse_normalize_* moments + pulse_rms_merge): the fp32 rows and their squares are
    exact in fp64, so the sums of n terms are off by at most n u64 sum|x| and n u64 sum x^2 (deterministic bound, any order); then the
    batch mean / variance and the merge, a few u64 per operation.  _merge64's own fp64 evaluation obeys the same bound: twice it."""
    x = f64(x)
    n = x.shape[0]
    tot = count + n
    e_s, e_q = n * U64 * x.abs().sum(0), n * U64 * (x * x).sum(0)
    bm = x.mean(0)
    q = (x * x).sum(0)
    e_bm = e_s / n + U64 * bm.abs()
    bv = x.var(0, unbiased=True)
    e_bv = (e_q + 2 * n * bm.abs() * e_bm + 4 * U64 * (q + n * bm * bm)) / (n - 1)
    delta = bm - mean
    e_mean = e_bm * n / tot + 4 * U64 * (mean.abs() + delta.abs() * n / tot)
    m2 = var * count + bv * n + delta * delta * count * n / tot
    e_var = (e_bv * n + 2 * delta.abs() * e_bm * count * n / tot + 8 * U64 * m2) / tot + U64 * m2 / tot
    return 2 * e_mean, 2 * e_var


def merge_chain64(mean, var, count, batches):
    """_merge64 over consecutive batches from fp64 (mean, var, count), with the bound of each merge (_merge64_tol) and the propagated
    bound of the statistics it starts from: (mean, (tol of mean), var, (tol of var), count)."""
    tm, tv = torch.zeros_like(mean), torch.zeros_like(var)
    for x in batches:
        n = x.shape[0]
        tot = count + n
        delta = f64(x).mean(0) - mean
        em, ev = _merge64_tol(mean, var, count, x)
        tv = tv * count / tot + 2 * delta.abs() * count * n / tot ** 2 * tm + ev
        tm = tm * count / tot + em
        mean, var, count, _, _ = _merge64(mean, var, count, x)
    return mean, tm, var, tv, count


def check_rms(rep, link, rms, start, batches):
    """A RunningMeanStdB200's fp64 state after merging `batches` into start = (mean, var, count): mean and var within the chained fp64
    summation bound, the count exact."""
    mean, tm, var, tv, count = merge_chain64(*start, batches)
    check(rep, f"{link} running_mean", rms.running_mean, mean, tm)
    check(rep, f"{link} running_var", rms.running_var, var, tv)
    check_exact(rep, f"{link} count", rms.count.reshape(1), torch.tensor([float(count)], dtype=torch.float64, device=rms.count.device))


def rms_f32(mean, var, count, batches):
    """The fp32 mean / rstd the kernels normalise with after merging `batches` into fp64 (mean, var, count)."""
    for x in batches:
        mean, var, count, _, _ = _merge64(mean, var, count, x)
    return mean.float(), 1.0 / torch.sqrt(var.float() + 1e-5)


def _check_normalized(rep, link, out, x, mean32, rstd32, cols, one_col, slack=0.0, clamp=5.0):
    y, tol = normalize_ref(x, mean32, rstd32, clamp)
    check(rep, link, out[:, :cols], y, tol + slack * y.abs())
    _check_pads(rep, link, out, one_col + 1 if one_col is not None else cols, one_col)


def check_split(rep, P, T, obs, mean32, rstd32, E, S, slack=0.0):
    """pulse_normalize_split's two operands: P[:, E:] = [self | 1 | 0...], T = [traj + heights | 1 | 0...] (P[:, :E] is not its)."""
    m, r = mean32.reshape(-1), rstd32.reshape(-1)
    _check_normalized(rep, "split normalise P self window (bf16)", P[:, E:], obs[:, :S], m[:S], r[:S], S, S, slack)
    Tn = obs.shape[1] - S
    _check_normalized(rep, "split normalise T task (bf16)", T, obs[:, S:], m[S:], r[S:], Tn, Tn, slack)


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


def check_ppo_loss(rep, pol, M, actions, old_nlp, adv, ret, mus):
    """pulse_ppo_loss on the kernel's own mu / value (the actor's and critic's training heads): dmu, dv, the statistics; the rows must
    cover every clip regime and |mu| > 1."""
    b = pol._buf(M, True)
    A = pol.A
    dmu, dv = b["dmu"], b["dv"]
    mu, value = pol.actor._ws[(M, True)]["out"][:M], pol.critic._ws[(M, True)]["out"][:M]
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
    check(rep, "ppo_loss dmu (bf16)", dmu[:M, :A], ref["dmu"], tol_mu)
    rep.rows[-1] = rep.rows[-1][:3] + (f"{n_amb} of {M} rows",)
    _check_pads(rep, "ppo_loss dmu", dmu[:M], A)
    check(rep, "ppo_loss dv (bf16)", dv[:M, 0], ref["dv"], ref["tol_v"])
    _check_pads(rep, "ppo_loss dv", dv[:M], 1)
    st = pol.stats.double()
    dev = st.device
    for k, name in enumerate(("sum a_loss", "sum c_loss", "sum b_loss", "sum kl", "clipped rows", "sum neglogp")):
        check(rep, f"ppo_loss stats[{k}] {name}", st[k:k + 1], ref["stats"][k].reshape(1), torch.as_tensor(ref["stats_tol"][k], dtype=torch.float64,
                                                                                                           device=dev).reshape(1) + 1e-300)
    return n_amb


def check_disc(rep, pol, B, snap, disc_stats, amp, slot=0):
    """The discriminator chain of one minibatch from operand slot `slot`: the normalised AMP batches (each with the statistics merged up
    to the batch before it, starting from disc_stats = (mean, var, count) in fp64), the forward / backward links, disc_loss, the
    gradient-penalty chain and the weight-gradient totals with the regulariser terms."""
    disc = pol.disc
    L1, L2, L3 = disc.mlp.layers
    db = disc._buf(B)
    xd = db["x"][slot]
    dev = xd.device
    mean, var, cnt = disc_stats
    for k, src in enumerate(amp):     # each batch is normalised with the statistics merged up to the batch before it
        m32, r32 = mean.float(), 1.0 / torch.sqrt(var.float() + 1e-5)
        _check_normalized(rep, f"disc normalised batch {k} (bf16)", xd[k * B:(k + 1) * B], src, m32, r32, L1.K, L1.K, slack=4 * U32)
        mean, var, cnt, _, _ = _merge64(mean, var, cnt, src)
    wd, bd = check_mlp(rep, "disc", disc.mlp, snap, xd, db["dlogit"], 3 * B)
    wsd = disc.mlp._ws[(3 * B, True)]
    gl, tl, dstats, dstats_tol = disc_loss_ref(wsd["out"][:3 * B], 2 * B, disc.disc_coef)
    check(rep, "disc_loss dlogit (bf16)", db["dlogit"][:3 * B, 0], gl, tl)
    _check_pads(rep, "disc_loss dlogit", db["dlogit"], 1)
    sd = disc.stats.double()
    for k in range(4):
        check(rep, f"disc_loss stats[{k}]", sd[k:k + 1], dstats[k].reshape(1).to(dev),
              torch.as_tensor(dstats_tol[k], dtype=torch.float64, device=dev).reshape(1) + 1e-300)
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
        reg = torch.zeros(l.N, l.Kp, dtype=torch.float64, device=dev)
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
