"""Development tool: per-phase clock trace of CTA 0 of one GEMM launch.  Needs the trace build:
    tools/build_variant.sh trace gemm_wgmma.cu -DPULSE_GEMM_VARIANT=3
    PULSE_ALT_LIB=$PWD/pulse_b200/build/libpulse_trace.so python tools/gemm_trace.py"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulse_b200 import _lib  # noqa: E402
_lib.LIB_PATH = os.environ["PULSE_ALT_LIB"]
from pulse_b200.dense import gemm  # noqa: E402

NAMES = {0: "start", 1: "setup done", 2: "producer past griddep wait", 3: "first stage landed", 4: "item0 MMAs retired", 16: "epi item0 staged",
         17: "epi item0 done", 5: "item1 MMAs retired", 18: "epi item1 staged", 19: "epi item1 done", 6: "item2 MMAs retired",
         20: "epi item2 staged", 21: "epi item2 done", 10: "teardown"}


def main():
    dev = torch.device("cuda:0")
    lib = _lib.load()
    lib.pulse_debug_gemm_trace.argtypes = [C.c_void_p]
    bf = lambda r, c: (torch.randn(r, c, device=dev) * 0.1).bfloat16()
    for name, (M, N, K, kw) in {
        "fwd1 relu M16384 N1024 K960": (16384, 1024, 960, dict(act="relu", bias=True)),
        "fwd2 relu M16384 N512 K1024": (16384, 512, 1024, dict(act="relu", bias=True)),
        "fwd silu+preact M16384 N1536 K960": (16384, 1536, 960, dict(act="silu", bias=True, preact=True)),
        # the production input-gradient GEMMs: actor / critic dgrad of layer 1 (ReLU bit-word gate) and the gradient penalty's G
        "dgrad gate_mask M16384 N1024 K512": (16384, 1024, 512, dict(dgrad=True, gate_mask=True)),
        "dgrad alpha+sumsq M4096 N1960 K1024": (4096, 1960, 1024, dict(dgrad=True, alpha=0.01, sumsq=True)),
    }.items():
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        if kw.get("dgrad"):   # A = dY [M, K], B = W [K, N] read MN-major
            a, b = bf(M, K), bf(K, N)
            args = dict(out=out, b_mn=True)
            if kw.get("gate_mask"):
                args["gate_mask"] = torch.randint(-2**31, 2**31 - 1, ((N + 31) // 32, M), device=dev, dtype=torch.int32)
            if kw.get("alpha"):
                args["alpha"] = kw["alpha"]
            if kw.get("sumsq"):
                args["sumsq"] = torch.zeros(1, device=dev, dtype=torch.float64)
        else:
            a, b = bf(M, K), bf(N, K)
            args = dict(out=out, act=kw["act"], bias=torch.zeros(N, device=dev))
            if kw.get("preact"):
                args["preact"] = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        for _ in range(3):
            gemm(a, b, **args)
        torch.cuda.synchronize()
        buf = (C.c_longlong * 32)()
        lib.pulse_debug_gemm_trace(buf)
        t0 = buf[0]
        print(f"--- {name}")
        for slot, t in sorted(((s, buf[s]) for s in NAMES if buf[s] >= t0), key=lambda x: x[1]):
            print(f"   {t - t0:8d} cyc  {NAMES[slot]}")


if __name__ == "__main__":
    main()
