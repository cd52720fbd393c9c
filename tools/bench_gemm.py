"""GEMM micro-benchmark: wgmma kernel vs torch.matmul (cuBLAS) at the MLP shapes."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulse_b200.dense import gemm_nt  # noqa: E402


def t(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    dev = torch.device("cuda:0")
    res = []
    for (M, N, K) in [(16384, 1024, 960), (16384, 512, 1024), (16384, 128, 512), (16384, 1024, 1984), (1024, 960, 16384), (8192, 8192, 8192)]:
        a = torch.randn(M, K, device=dev).bfloat16()
        b = torch.randn(N, K, device=dev).bfloat16()
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        bias = torch.zeros(N, device=dev)
        ms = t(lambda: gemm_nt(a, b, bias=bias, act="relu", out=out))
        ms_t = t(lambda: torch.relu(torch.nn.functional.linear(a, b)))
        fl = 2.0 * M * N * K
        res.append({"M": M, "N": N, "K": K, "ms": ms, "tflops": fl / ms / 1e9, "torch_ms": ms_t, "torch_tflops": fl / ms_t / 1e9})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
