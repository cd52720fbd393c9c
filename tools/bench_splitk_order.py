"""Cost of the fixed-order split-K reduction: the update's weight-gradient GEMMs timed inside CUDA graphs, once through dense.gemm
(every split writes a slab, pulse_ordered_sum_add adds the slabs in split order) and once with the slices' bulk reductions added in
place (scheduling-dependent order).  usage: python tools/bench_splitk_order.py"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulse_b200 import _lib, dense  # noqa: E402
from pulse_b200.nets import pick_split  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
torch.manual_seed(0)
print(torch.cuda.get_device_name(0))
tot_slab = tot_inplace = 0.0
# weight-gradient GEMMs of one PPO minibatch: (out rows N, out cols Kp, reduction rows M) for actor / critic / disc layers
shapes = [(1024, 960, 16384), (512, 1088, 16384), (69, 576, 16384), (1024, 960, 16384), (512, 1088, 16384),
          (1024, 1984, 12288), (512, 1088, 12288), (1024, 1984, 4096), (512, 1088, 4096)]
for (N, Kp, M) in shapes:
    dy = (torch.randn(M, (N + 7) // 8 * 8, device=dev) * 0.1).bfloat16()[:, :N]
    x = torch.randn(M, Kp, device=dev).bfloat16()
    out = torch.zeros(N, Kp, device=dev)
    s = pick_split(((N + 127) // 128) * ((Kp + 127) // 128), (M + 63) // 64)
    def slab():
        dense.gemm(dy, x, a_mn=True, b_mn=True, out_f32=out, accumulate=True, split_k=s)
    def inplace():
        ep = _lib.GemmEpilogue(); ep.alpha = 1.0; ep.out_f32 = out.data_ptr(); ep.ldf = out.stride(0); ep.accumulate = 1
        _lib.check(lib.pulse_gemm_bf16(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), N, Kp, M, C.byref(ep), s,
                                       _lib.GEMM_A_MN | _lib.GEMM_B_MN, _lib.current_stream(dev)), "gemm")
    res = {}
    graphs = {}
    for name, fn in (("slab", slab), ("inplace", inplace)):
        for _ in range(3): fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(20): fn()
        graphs[name] = g
    for name in ("slab", "inplace", "slab", "inplace"):
        graphs[name].replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(5): graphs[name].replay()
        b.record(); torch.cuda.synchronize()
        res.setdefault(name, []).append(a.elapsed_time(b) / 100 * 1e3)
    sl, ip = min(res["slab"]), min(res["inplace"])
    tot_slab += sl; tot_inplace += ip
    print(f"N {N} Kp {Kp} M {M} split {s}: slab {sl:.1f} us  in-place {ip:.1f} us")
print(f"sum slab {tot_slab:.1f} us  in-place {tot_inplace:.1f} us  per minibatch set (CUDA graphs)")
