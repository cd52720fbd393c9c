"""Every NON-GEMM kernel of one PPO + discriminator minibatch update, timed alone (CUDA events, back-to-back launches) with its HBM floor.

    python tools/bench_update_misc.py [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulse_b200 import _lib  # noqa: E402
if os.environ.get("PULSE_ALT_LIB"):
    _lib.LIB_PATH = os.environ["PULSE_ALT_LIB"]
from pulse_b200.ppo import PPOPolicy  # noqa: E402


def timed(fn, reps=20, iters=10):
    """GPU time per call: `reps` calls captured into one CUDA graph (no Python between the launches), replayed `iters` times."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / (iters * reps) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    hbm = 3350.0   # fallback: H100 SXM data sheet HBM3 bandwidth
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        hbm = json.load(open(p)).get("hbm_gbs", hbm)
    lib = _lib.load()
    st = lambda: _lib.current_stream(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    M, B = 16384, 4096
    pol = PPOPolicy(device=dev, seed=0, with_disc=True)
    obs = torch.randn(M, 934, device=dev, generator=g)
    act = torch.randn(M, 69, device=dev, generator=g) * 0.1
    mu = torch.randn(M, 69, device=dev, generator=g) * 0.1
    nlp = torch.randn(M, device=dev, generator=g) + 60
    adv, ret = torch.randn(M, device=dev, generator=g), torch.randn(M, device=dev, generator=g)
    amp = tuple(torch.randn(B, 1960, device=dev, generator=g) for _ in range(3))
    for _ in range(2):
        pol.train_minibatch(obs, act, nlp, adv, ret, old_mu=mu, amp=amp)     # allocates every workspace
    torch.cuda.synchronize()
    rows = []

    def case(name, fn, nbytes):
        us = timed(fn)
        rows.append({"name": name, "us": round(us, 2), "floor_us": round(nbytes / hbm / 1e3, 2), "gbs": round(nbytes / us / 1e3, 1)})
        print(f"{name:34s} {us:8.2f} us   floor {nbytes / hbm / 1e3:6.2f} us   {nbytes / us / 1e3:8.1f} GB/s")

    bx = pol._buf(M, True)
    case("obs normalize_update (+merge)", lambda: pol.obs_rms.normalize_update(obs, bx["x2"][0]), M * 934 * 4 + M * pol.Kp * 2)
    case("obs normalize_into", lambda: pol.obs_rms.normalize_into(obs, bx["x2"][0]), M * 934 * 4 + M * pol.Kp * 2)
    bd = pol.disc._buf(B)
    case("amp normalize_update x3 (+merge)", lambda: [pol.disc.rms.normalize_update(s_, bd["x"][0][k * B:(k + 1) * B]) for k, s_ in enumerate(amp)],
         3 * (B * 1960 * 4 + B * pol.disc.Kp * 2))
    ws = pol.critic._ws[(M, True)]
    h2, dh = ws["act"][1], ws["dact"][1]
    head = pol.critic.layers[-1]
    case("head1_forward (critic)", lambda: pol.critic.forward(bx["x2"][0], train=True) if False else _lib.check(lib.pulse_head1_forward(
        h2.data_ptr(), h2.stride(0), M, head.Kp, head.w_bf16.data_ptr(), pol.critic._zero_bias().data_ptr(), ws["out"].data_ptr(), ws["out"].stride(0), st()), "h1f"),
         M * head.Kp * 2)
    case("head1_backward (critic)", lambda: pol.critic._backward_head(ws, bx["dv"], M), 2 * M * head.Kp * 2)
    args = _lib.PpoLossArgs(mu=mu.data_ptr(), ld_mu=69, value=ws["out"].data_ptr(), ld_value=ws["out"].stride(0), actions=act.data_ptr(),
                            old_neglogp=nlp.data_ptr(), advantages=adv.data_ptr(), returns=ret.data_ptr(), old_mu=mu.data_ptr(),
                            logstd=pol.logstd.data_ptr(), num_actions=69, e_clip=0.2, critic_coef=5.0, bounds_coef=10.0, dmu=bx["dmu"].data_ptr(),
                            ld_dmu=bx["dmu"].stride(0), dvalue=bx["dv"].data_ptr(), ld_dv=bx["dv"].stride(0), stats=pol.stats.data_ptr())
    case("ppo_loss", lambda: _lib.check(lib.pulse_ppo_loss(C.byref(args), M, st()), "ppo"), M * 69 * 4 * 3 + M * 72 * 2 + M * 20)
    n = pol.flat.numel
    case("sum_squares (grad norm)", lambda: _lib.check(lib.pulse_sum_squares(pol.flat.grads.data_ptr(), n, pol.flat.sumsq.data_ptr(), st()), "ss"), n * 4)
    case("adam_step (self-contained)", lambda: pol.flat.adam_step(2e-5, max_norm=0.0), n * (4 * 4 + 3 * 4 + 2 + 4))
    case("grads memset", lambda: pol.flat.grads.zero_(), n * 4)
    dw = pol.disc
    L1, L2, L3 = dw.mlp.layers

    def reg():
        r = _lib.WeightReg()
        r.count = 3
        for k, l in enumerate((L1, L2, L3)):
            blk = r.block[k]
            blk.w, blk.g, blk.rows, blk.cols, blk.ld, blk.coef = l.weight.data_ptr(), l.weight_grad.data_ptr(), l.N, l.K, l.Kp, 1e-3
            blk.sumsq = dw.stats[6:].data_ptr()
        _lib.check(lib.pulse_weight_reg(C.byref(r), st()), "reg")
    case("weight_reg (disc decay + sums)", reg, (L1.N * L1.K + L2.N * L2.K + L3.K) * 12)
    dws = dw.mlp._ws[(3 * B, True)]
    h2d = dws["act"][1][2 * B:]
    case("relu_mask_scale", lambda: _lib.check(lib.pulse_relu_mask_scale(h2d.data_ptr(), h2d.stride(0), B, L2.N, L3.weight.data_ptr(), bd["g2"].data_ptr(),
                                                                        bd["g2"].stride(0), st()), "rms"), B * L2.N * 4)
    lg = dws["out"]
    case("disc_loss", lambda: _lib.check(lib.pulse_disc_loss(lg.data_ptr(), lg.stride(0), 2 * B, B, 5.0, bd["dlogit"].data_ptr(), bd["dlogit"].stride(0),
                                                            dw.stats.data_ptr(), st()), "dl"), 3 * B * 6)
    tot = sum(r["us"] for r in rows)
    print(f"sum {tot:.1f} us, floor {sum(r['floor_us'] for r in rows):.1f} us")
    if a.json:
        json.dump({"cases": rows, "sum_us": tot}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
