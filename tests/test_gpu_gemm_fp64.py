"""pulse_gemm_bf16 cell by cell against float64 (tests/gemm_fp64.py): every case in both operand families -- exact integers (outputs bit
for bit: fp32 values, bf16 round-to-nearest-even, mask bits y > 0) and random normal (the Gemm rounding bound) -- under the default
dispatch, PULSE_GEMM_STAGES=4 and PULSE_GEMM_BN=128.  After every launch pulse_gemm_last_launch must report the kernel the dispatch model
predicts for the case, every output is checked inside guard bands, split-K slabs one by one, and the slab cases' ordered_sum_add /
column_sum_add bit for bit against the host sum in the kernel's order.  A last test asserts that the run reached every row of
gemm_fp64.CELLS; PULSE_GEMM_SMS, read once per process, is covered by a child process at 1 and 7 SMs.
Run with -s to print every case's cells and the err / tol of each link.
"""
import ctypes as C
import os
import subprocess
import sys
import time

import pytest
import torch

from pulse_b200 import _lib
from tests import gemm_fp64 as gf
from tests.fp64_ref import Report, check_exact

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = gf.all_cases()
REACHED = {}              # CELLS row -> the first case that reached it and passed
STATS = {"cases": 0, "launches": 0, "ties": 0, "t0": None}


def _sms() -> int:
    n = torch.cuda.get_device_properties(DEV).multi_processor_count
    e = os.environ.get("PULSE_GEMM_SMS")
    return int(e) if e is not None and 1 <= int(e) < n else n


def launch(c: gf.Case, ops: gf.Operands, outs: gf.Outputs) -> None:
    """One pulse_gemm_bf16 call through the raw ABI, or dense.gemm for its accumulate + split route (slabs, then the ordered sum)."""
    if c.f32 == "dense":
        from pulse_b200.dense import gemm
        gemm(ops.A, ops.B, a_mn=c.a_mn, b_mn=c.b_mn, out_f32=outs.f32.view, accumulate=True, split_k=c.split_k)
        return
    ep = _lib.GemmEpilogue()
    ep.alpha = c.alpha
    ep.act = {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "silu": _lib.ACT_SILU}[c.act]
    if ops.bias is not None:
        ep.bias = ops.bias.data_ptr()
    if c.gate in ("relu", "silu"):
        ep.gate, ep.ldg = ops.gate.data_ptr(), ops.gate.stride(0)
        ep.gate_mode = _lib.ACT_RELU if c.gate == "relu" else _lib.ACT_SILU
    if c.gate == "bits":
        ep.gate_mask, ep.ld_gmask = ops.gate_words.data_ptr(), ops.gate_words.stride(0)
    for name, ptr_f, ld_f in (("out", "out", "ldo"), ("out_t", "out_t", "ldot"), ("preact", "preact", "ldp")):
        g = getattr(outs, name)
        if g is not None:
            setattr(ep, ptr_f, g.view.data_ptr())
            setattr(ep, ld_f, g.view.stride(0))
    if outs.f32 is not None:
        ep.out_f32 = outs.f32.view.data_ptr()
        if c.f32 == "slabs":
            ep.split_stride, ep.ldf = outs.f32.view.stride(0), outs.f32.view.stride(1)
        else:
            ep.ldf = outs.f32.view.stride(0)
        ep.accumulate = int(c.f32 == "accum")
    if outs.colsum is not None:
        ep.colsum = outs.colsum.view.data_ptr()
    if outs.sumsq is not None:
        ep.sumsq = outs.sumsq.view.data_ptr()
    if outs.mask is not None:
        ep.relu_mask, ep.ld_rmask = outs.mask.view.data_ptr(), outs.mask.view.stride(0)
    flags = (_lib.GEMM_A_MN if c.a_mn else 0) | (_lib.GEMM_B_MN if c.b_mn else 0)
    _lib.check(_lib.load().pulse_gemm_bf16(ops.A.data_ptr(), ops.A.stride(0), ops.B.data_ptr(), ops.B.stride(0), c.M, c.N, c.K,
                                           C.byref(ep), c.split_k, flags, _lib.current_stream(DEV)), "pulse_gemm_bf16")


def run_case(c: gf.Case, setenv, variants=tuple(gf.VARIANTS), verbose: bool = True) -> None:
    """c in both families under each variant (setenv(name, value or None) sets the dispatch overrides).  Records the CELLS rows the
    launches reached once the case has passed."""
    from pulse_b200.dense import column_sum_add, ordered_sum_add
    sms = _sms()
    reached = []
    for exact in (True, False):
        ops = gf.Operands(c, exact, DEV)
        ref = gf.Expected(c, ops)
        if exact and c.out and ref.exact:
            q = ref.v.abs()
            STATS["ties"] += int(((q > 256) & (q < 512) & (torch.remainder(q, 2) == 1)).sum())
        for v in variants:
            for key in ("PULSE_GEMM_STAGES", "PULSE_GEMM_BN"):
                setenv(key, gf.VARIANTS[v].get(key))
            rep = Report(f"{c.name} [{'exact' if exact else 'bounded'}, {v}]")
            outs = gf.Outputs(c, ops, DEV)
            launch(c, ops, outs)
            got = _lib.gemm_last_launch()
            slabs_sum = None
            if c.f32 == "slabs":
                ns = gf.num_splits(c.K, c.split_k)
                slabs = outs.f32.view[:ns]
                total = torch.zeros(c.M, c.N, device=DEV)
                ordered_sum_add(slabs, total)
                cs = torch.zeros(c.N, device=DEV)
                column_sum_add(slabs[0], cs)
                torch.cuda.synchronize()
                slabs_sum = (total, gf.ordered_sum_host(slabs, torch.zeros(c.M, c.N, device=DEV)))
                check_exact(rep, "column_sum_add (64-row chunks, then the chunks)", cs, gf.column_sum_host(slabs[0], torch.zeros(c.N, device=DEV)))
            torch.cuda.synchronize()
            gf.check_outputs(rep, c, ops, outs, ref, slabs_sum=slabs_sum)
            want = gf.predict(c, sms, v)
            assert got == want, f"{c.name} [{v}]: the launch took {got}, the dispatch model predicts {want}"
            STATS["launches"] += 1
            reached += [(cid, v) for cid in gf.cells_of(c, got, v)]
            if verbose:
                print(f"\n{gf.cell_name(c, got)}  grid {got['grid']} splits {got['splits']}\n" + rep.text())
    for cid, v in reached:
        REACHED.setdefault(cid, f"{c.name} [{v}]")
    for key in ("PULSE_GEMM_STAGES", "PULSE_GEMM_BN"):
        setenv(key, None)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_gemm_cell_fp64(monkeypatch, case):
    if STATS["t0"] is None:
        STATS["t0"] = time.time()

    def setenv(key, value):
        if value is None:
            monkeypatch.delenv(key, raising=False)
        else:
            monkeypatch.setenv(key, value)

    run_case(case, setenv)
    STATS["cases"] += 1


def test_every_cell_reached():
    """Every row of gemm_fp64.CELLS was reached by a case that passed, and the exact family produced bf16 rounding ties above 256."""
    if STATS["cases"] < len(CASES):
        pytest.skip("needs the whole case list of test_gemm_cell_fp64 in this session")
    if torch.cuda.get_device_properties(DEV).multi_processor_count != gf.H100_SMS:
        pytest.skip("the cell list is written for an H100's 132 SMs")
    missing = [cid for cid, _ in gf.CELLS if cid not in REACHED]
    print(f"\n{len(CASES)} cases, {STATS['launches']} launches in {time.time() - STATS['t0']:.1f} s; {STATS['ties']} bf16 ties above 256")
    for cid, _ in gf.CELLS:
        print(f"  {cid:<58s} {REACHED.get(cid, 'NOT REACHED')}")
    assert missing == []
    assert STATS["ties"] > 0


CHILD = """
import os, sys
sys.path.insert(0, {root!r})
from tests import gemm_fp64 as gf
from tests.test_gpu_gemm_fp64 import run_case, REACHED
def setenv(key, value):
    if value is None:
        os.environ.pop(key, None)
    else:
        os.environ[key] = value
cases = gf.table_cases() + gf.persistent_cases()
for c in cases:
    run_case(c, setenv, variants=("default",), verbose=False)
print("cases", len(cases), "cells", len(REACHED))
"""


@pytest.mark.parametrize("sms", [1, 7])
def test_gemm_cells_on_few_sms(sms):
    """PULSE_GEMM_SMS is read once per process: the table and persistent-grid cases in a child process on 1 and 7 SMs, where hundreds
    of items pass through one CTA's ring and small shapes reach the wide tile."""
    env = dict(os.environ, PULSE_GEMM_SMS=str(sms))
    env.pop("PULSE_GEMM_STAGES", None)
    env.pop("PULSE_GEMM_BN", None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD.format(root=ROOT)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    print(f"\nPULSE_GEMM_SMS={sms}: {r.stdout.strip()}")
