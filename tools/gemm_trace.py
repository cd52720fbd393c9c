"""Development tool: per-phase clock trace of CTA 0 of one GEMM launch, with the ring-barrier stall counters.  Needs the trace build:
    tools/build_variant.sh trace gemm_wgmma.cu -DPULSE_GEMM_VARIANT=3
    PULSE_ALT_LIB=$PWD/pulse_b200/build/libpulse_trace.so python tools/gemm_trace.py [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulse_b200 import _lib  # noqa: E402
_lib.LIB_PATH = os.environ["PULSE_ALT_LIB"]
from pulse_b200.dense import gemm  # noqa: E402
from pulse_b200.nets import pick_split  # noqa: E402

NAMES = {0: "start", 1: "setup done", 2: "producer past griddep wait", 3: "first stage landed", 4: "item0 MMAs retired", 16: "epi item0 staged",
         17: "epi item0 done", 5: "item1 MMAs retired", 18: "epi item1 staged", 19: "epi item1 done", 6: "item2 MMAs retired",
         20: "epi item2 staged", 21: "epi item2 done", 10: "teardown"}
# value slots (not clocks since start): consumer warp 0's clocks waiting on `full` per item (22 + i), k-blocks per item (25 + i), producer
# clocks waiting on `empty` per item (28 + i), items 0..2 of CTA 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args_cli = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.load()
    lib.pulse_debug_gemm_trace.argtypes = [C.c_void_p]
    bf = lambda r, c: (torch.randn(r, c, device=dev) * 0.1).bfloat16()
    rows = []
    for name, (M, N, K, kw) in {
        "fwd1 relu M16384 N1024 K960": (16384, 1024, 960, dict(act="relu", bias=True)),
        "fwd2 relu M16384 N512 K1024": (16384, 512, 1024, dict(act="relu", bias=True)),
        "fwd silu+preact M16384 N1536 K960": (16384, 1536, 960, dict(act="silu", bias=True, preact=True)),
        # the production input-gradient GEMMs: actor / critic dgrad of layer 1 (ReLU bit-word gate) and the gradient penalty's G
        "dgrad gate_mask M16384 N1024 K512": (16384, 1024, 512, dict(dgrad=True, gate_mask=True)),
        "dgrad alpha+sumsq M4096 N1960 K1024": (4096, 1960, 1024, dict(dgrad=True, alpha=0.01, sumsq=True)),
        "disc fwd1 relu M12288 N1024 K1984": (12288, 1024, 1984, dict(act="relu")),
        "disc dgrad2 gate_mask M12288 N1024 K512": (12288, 1024, 512, dict(dgrad=True, gate_mask=True)),
        "gp du gate_mask M4096 N1024 K1960 (B K-major)": (4096, 1024, 1960, dict(dgrad=True, b_k_major=True, gate_mask=True)),
        # weight gradients of the update (A = dY^T, B = X^T, both MN-major; split-K as the nets pick it)
        "wgrad1 M1024 N934 K16384": (1024, 934, 16384, dict(wgrad=True)),
        "wgrad2 M512 N1024 K16384": (512, 1024, 16384, dict(wgrad=True)),
        "disc wgrad1 M1024 N1960 K12288": (1024, 1960, 12288, dict(wgrad=True)),
        "gp dW1 M1024 N1960 K4096": (1024, 1960, 4096, dict(wgrad=True)),
    }.items():
        if kw.get("wgrad"):
            Mp, Np = (M + 63) // 64 * 64, (N + 63) // 64 * 64
            a, b = bf(K, Mp)[:, :M], bf(K, Np)[:, :N]
            tiles = ((M + 127) // 128) * ((N + 127) // 128)
            args = dict(a_mn=True, b_mn=True, out_f32=torch.zeros(M, Np, device=dev), accumulate=True, split_k=pick_split(tiles, (K + 63) // 64))
        elif kw.get("dgrad"):   # A = dY [M, K], B = W [K, N] read MN-major
            out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
            a, b = bf(M, K), (bf(N, K) if kw.get("b_k_major") else bf(K, N))
            args = dict(out=out, b_mn=not kw.get("b_k_major"))
            if kw.get("gate_mask"):
                args["gate_mask"] = torch.randint(-2**31, 2**31 - 1, ((N + 31) // 32, M), device=dev, dtype=torch.int32)
            if kw.get("alpha"):
                args["alpha"] = kw["alpha"]
            if kw.get("sumsq"):
                args["sumsq"] = torch.zeros(1, device=dev, dtype=torch.float64)
        else:
            out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
            a, b = bf(M, K), bf(N, K)
            args = dict(out=out, act=kw["act"], bias=torch.zeros(N, device=dev) if kw.get("bias") else None)
            if kw.get("preact"):
                args["preact"] = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        for bn in ("128", "rule"):   # the 128 x 128 tile forced, then the width the shape rule picks
            trace_one(lib, f"{name} [{bn}]", bn, lambda: gemm(a, b, **args), rows)
    if args_cli.json:
        json.dump(rows, open(args_cli.json, "w"), indent=1)


def trace_one(lib, name, bn, run, rows):
    """one traced launch of run() with the 128 x 128 tile forced (bn = "128") or at the width the shape rule picks"""
    if bn == "128":
        os.environ["PULSE_GEMM_BN"] = "128"
    else:
        os.environ.pop("PULSE_GEMM_BN", None)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    buf = (C.c_longlong * 32)()
    lib.pulse_debug_gemm_trace(buf)
    t0 = buf[0]
    print(f"--- {name}")
    for slot, t in sorted(((s, buf[s]) for s in NAMES if buf[s] >= t0), key=lambda x: x[1]):
        print(f"   {t - t0:8d} cyc  {NAMES[slot]}")
    # second item: from the end of item 0's epilogue to its own MMAs retiring (first item, from its first stage landing, when CTA 0
    # has only one; the kernel clears the slots at launch)
    i = 1 if buf[5] > 0 else 0
    main_loop = buf[5] - buf[17] if i else buf[4] - buf[3]
    kb, full = buf[25 + i], buf[22 + i]
    r = {"name": name, "item_index": i, "kb": kb, "main_loop": main_loop, "clk_per_kb": round(main_loop / max(kb, 1)),
         "full_wait": full, "full_share": round(full / max(main_loop, 1), 3), "empty_wait": buf[28 + i],
         "full_wait_items": [buf[22], buf[23], buf[24]], "empty_wait_items": [buf[28], buf[29], buf[30]]}
    rows.append(r)
    print(f"   item{i}: {kb} k-blocks, main loop {main_loop} clk ({r['clk_per_kb']}/k-block), consumer waits on full {full} clk "
          f"({100 * r['full_share']:.0f} %), producer waits on empty {buf[28 + i]} clk")


if __name__ == "__main__":
    main()
