"""Every GEMM of one PPO + discriminator minibatch update, timed alone (CUDA events, warm L2), with its tensor / HBM floor, at the tile
width the shape rule picks and with the 128 x 128 tile forced (PULSE_GEMM_BN=128).
The epilogue arguments are the ones the update passes: the nets are bias-augmented (no bias vector, no column sums), the forward
layers write ReLU mask words and the input-gradient GEMMs are gated by them.

    python tools/bench_update_gemms.py [--json out.json]
floor_us = max(flops / bf16 peak, compulsory bytes / HBM peak) from MEASURED_PEAKS.json (sustained figures).
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulse_b200 import _lib  # noqa: E402
if os.environ.get("PULSE_ALT_LIB"):      # A/B a differently built library on the same box
    _lib.LIB_PATH = os.environ["PULSE_ALT_LIB"]
from pulse_b200.dense import gemm  # noqa: E402
from pulse_b200.nets import pad_k, pick_split  # noqa: E402


def timed(fn, iters=30, warm=5):
    for _ in range(warm):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--only", default=None, help="run just the cases whose name contains this (for ncu captures)")
    ap.add_argument("--vae", action="store_true", help="the SiLU stacks of the PULSE VAE (im_z_fit.yaml) instead of the PPO nets")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    peaks = {"bf16": 989.0, "hbm": 3350.0}   # fallback: H100 SXM data sheet (dense bf16 TFLOP/s, HBM3 GB/s)
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        peaks = {"bf16": d.get("bf16_tflops_sustained", d.get("bf16_tflops", peaks["bf16"])), "hbm": d.get("hbm_gbs", peaks["hbm"])}
    bf = lambda r, c: (torch.randn(r, c, device=dev) * 0.1).bfloat16()
    rows = []

    def case(name, M, N, K, kind, gate=None, colsum=False, f32=False, bf16_out=True, alpha=1.0, act="relu", preact=False, bias=False,
             relu_mask=False, sumsq=False):
        """kind: 'nt' (A [M,K], B [N,K]), 'dgrad' (A [M,K], B [K,N] MN-major), 'wgrad' (A [K,M], B [K,N], atomics into fp32).
        gate: None, 'act' (bf16 saved tensor, act') or 'mask' (ReLU mask words); relu_mask: a forward case writes the mask words."""
        if a.only and a.only not in name:
            return
        Mp, Np, Kp = pad_k(M), pad_k(N), pad_k(K)
        kw = {}
        if kind == "nt":
            A, B = bf(M, Kp), bf(Np, Kp)
            av, bv = A, B[:N]
        elif kind == "dgrad":
            A, B = bf(M, Kp), bf(Kp, Np)
            av, bv = A[:, :K], B[:K, :N]
            kw.update(b_mn=True)
        else:
            A, B = bf(K, Mp), bf(K, Np)
            av, bv = A[:, :M], B[:, :N]
            kw.update(a_mn=True, b_mn=True)
        byt = av.numel() * 2 + bv.numel() * 2
        if kind == "wgrad":
            tiles = ((M + 127) // 128) * ((N + 127) // 128)
            kw.update(out_f32=torch.zeros(M, Np, device=dev), accumulate=True, split_k=pick_split(tiles, (K + 63) // 64))
            byt += M * N * 4 * 2
        else:
            if bf16_out:
                kw.update(out=torch.zeros(M, Np, device=dev, dtype=torch.bfloat16))
                byt += M * N * 2
            if f32:
                kw.update(out_f32=torch.zeros(M, Np, device=dev))
                byt += M * N * 4
            if kind == "nt" and gate is None:
                kw.update(act=act if bf16_out and not f32 else None)
                if bias:
                    kw.update(bias=torch.zeros(N, device=dev))
                if preact:
                    kw.update(preact=torch.zeros(M, Np, device=dev, dtype=torch.bfloat16))
                    byt += M * N * 2
                if relu_mask:
                    kw.update(relu_mask=torch.zeros((N + 31) // 32, M, device=dev, dtype=torch.int32))
                    byt += M * N // 8
        if gate == "act":
            kw.update(gate=bf(M, Np), gate_mode=act)
            byt += M * N * 2
        elif gate == "mask":
            kw.update(gate_mask=torch.randint(-2 ** 31, 2 ** 31 - 1, ((N + 31) // 32, M), device=dev, dtype=torch.int32))
            byt += M * N // 8
        if sumsq:
            kw.update(sumsq=torch.zeros(1, device=dev, dtype=torch.float64))
        if colsum:
            kw.update(colsum=torch.zeros(Np, device=dev))
        if alpha != 1.0:
            kw.update(alpha=alpha)
        os.environ["PULSE_GEMM_BN"] = "128"   # the 128 x 128 tile, then the width the shape rule picks
        us128 = timed(lambda: gemm(av, bv, **kw))
        del os.environ["PULSE_GEMM_BN"]
        us = timed(lambda: gemm(av, bv, **kw))
        fl = 2.0 * M * N * K
        floor = max(fl / peaks["bf16"] / 1e6, byt / peaks["hbm"] / 1e3)
        rows.append({"name": name, "M": M, "N": N, "K": K, "kind": kind, "us": round(us, 2), "us_bn128": round(us128, 2), "tflops": round(fl / us / 1e6, 1),
                     "gbs": round(byt / us / 1e3, 1), "floor_us": round(floor, 2), "eff": round(floor / us, 3)})

    B, Bd, Bg = 16384, 12288, 4096
    if a.vae:
        for net, sizes in (("enc", [934, 1536, 1024, 512, 160]), ("prior", [358, 1536, 1024, 512]), ("dec", [390, 3096, 2048, 1024])):
            for i in range(len(sizes) - 1):
                k, n = sizes[i], sizes[i + 1]
                case(f"{net}.fwd{i}", B, n, k, "nt", act="silu", preact=True, bias=True)
                case(f"{net}.wgrad{i}", n, k, B, "wgrad")
                if i > 0:
                    case(f"{net}.dgrad{i}", B, k, n, "dgrad", gate="act", colsum=True, act="silu")
    for net, head in (() if a.vae else (("actor", 69), ("critic", 1))):
        case(f"{net}.fwd1", B, 1024, 934, "nt", relu_mask=True)
        case(f"{net}.fwd2", B, 512, 1024, "nt", relu_mask=True)
        case(f"{net}.head", B, head, 512, "nt", f32=True, bf16_out=False)
        case(f"{net}.wgrad_head", head, 512, B, "wgrad")
        case(f"{net}.dgrad_head", B, 512, head, "dgrad", gate="mask")
        case(f"{net}.wgrad2", 512, 1024, B, "wgrad")
        case(f"{net}.dgrad2", B, 1024, 512, "dgrad", gate="mask")
        case(f"{net}.wgrad1", 1024, 934, B, "wgrad")
    if a.vae:
        Bd = Bg = 0
    nonvae = lambda *args, **kw2: None if a.vae else case(*args, **kw2)
    nonvae("disc.fwd1", Bd, 1024, 1960, "nt", relu_mask=True)
    nonvae("disc.fwd2", Bd, 512, 1024, "nt", relu_mask=True)
    nonvae("disc.head", Bd, 1, 512, "nt", f32=True, bf16_out=False)
    nonvae("disc.wgrad_head", 1, 512, Bd, "wgrad")
    nonvae("disc.dgrad_head", Bd, 512, 1, "dgrad", gate="mask")
    nonvae("disc.wgrad2", 512, 1024, Bd, "wgrad")
    nonvae("disc.dgrad2", Bd, 1024, 512, "dgrad", gate="mask")
    nonvae("disc.wgrad1", 1024, 1960, Bd, "wgrad")
    nonvae("gp.g1", Bg, 1024, 512, "dgrad", gate="mask")
    nonvae("gp.G", Bg, 1960, 1024, "dgrad", alpha=0.01, sumsq=True)
    nonvae("gp.dW1", 1024, 1960, Bg, "wgrad")
    nonvae("gp.du", Bg, 1024, 1960, "nt", gate="mask")
    nonvae("gp.dW2", 512, 1024, Bg, "wgrad")
    nonvae("gp.dw3", Bg, 512, 1024, "nt", gate="mask", f32=True, bf16_out=False)
    tot, fl = sum(r["us"] for r in rows), sum(r["floor_us"] for r in rows)
    for r in rows:
        print(f"{r['name']:18s} {r['kind']:5s} M={r['M']:6d} N={r['N']:5d} K={r['K']:6d}  {r['us']:8.2f} us (128 x 128: {r['us_bn128']:8.2f})  {r['tflops']:7.1f} TF  "
              f"{r['gbs']:7.1f} GB/s  floor {r['floor_us']:7.2f} us  eff {r['eff']:.2f}")
    print(f"sum {tot:.1f} us (128 x 128 tiles: {sum(r['us_bn128'] for r in rows):.1f} us), floor {fl:.1f} us, eff {fl / tot:.3f}")
    if a.json:
        json.dump({"peaks": peaks, "cases": rows, "sum_us": tot, "floor_us": fl}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
