"""CPU checks of the AMP demo / replay rings: the numpy model of the device bookkeeping (tests/amp_buffers_model.py) against the
reference's ReplayBuffer and _store_replay_amp_obs run on the same draws (tests/golden/amp_buffers.npz), the permutation's
properties, the Philox index planes of the header's draw table, and the C layout of the new argument structs."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from tests import amp_buffers_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "amp_buffers.npz"))


def test_model_matches_reference_bookkeeping():
    res = M.run_script(M.RingModel(M.CAPACITY, M.SEED))
    branches = set()
    for s, (kind, rows, ctr, ids) in enumerate(res):
        np.testing.assert_array_equal(ctr, GOLDEN[f"s{s}_counters"], err_msg=f"step {s} counters")
        np.testing.assert_array_equal(ids, np.where(GOLDEN[f"s{s}_buffer"] == 0, -1, GOLDEN[f"s{s}_buffer"]), err_msg=f"step {s} buffer")
        if kind == "sample":
            prev_ids = res[s - 1][3] if s > 0 else None
            got = np.full(len(rows), -1) if (rows < 0).all() else prev_ids[rows]
            np.testing.assert_array_equal(got, GOLDEN[f"s{s}_ids"], err_msg=f"step {s} sampled rows")
        prev_ctr = res[s - 1][2] if s > 0 else np.zeros(5, np.int64)
        if kind == "sample":
            branches.add("empty" if prev_ctr[1] == 0 else ("mod_head" if prev_ctr[1] < M.CAPACITY else "full"))
            if ctr[3] > prev_ctr[3]:
                branches.add("rekey")
            if M.SCRIPT[s][1] > M.CAPACITY:
                branches.add("sample_wraps")
        else:
            if prev_ctr[0] + len(rows) > M.CAPACITY:
                branches.add("head_wrap")
            if prev_ctr[1] > M.CAPACITY:
                branches.add("keep_mask")
            if len(rows) == M.CAPACITY and M.SCRIPT[s][1] > M.CAPACITY:
                branches.add("subset")
    assert branches == {"empty", "mod_head", "full", "rekey", "sample_wraps", "head_wrap", "keep_mask", "subset"}


@pytest.mark.parametrize("m", [1, 2, 3, 5, 64, 100, 1000, 200000])
def test_feistel_is_a_permutation(m):
    p = M.permutation(M.SEED, M.PLANE_RING_PERM, 3, m)
    np.testing.assert_array_equal(np.sort(p), np.arange(m))
    if m >= 64:
        assert not np.array_equal(p, M.permutation(M.SEED, M.PLANE_RING_PERM, 4, m))   # a new key is a new permutation


def _header():
    return open(os.path.join(ROOT, "include", "pulse_b200.h")).read()


def test_ring_planes_distinct_and_in_draw_table():
    h = _header()
    planes = {k: int(v) for k, v in re.findall(r"#define PULSE_PLANE_([A-Z_]+) (\d+)", h)}
    assert planes == {"DEMO_CLIP": 5, "DEMO_TIME": 6, "REPLAY_KEEP": 7, "REPLAY_SUBSET": 8, "RING_PERM": 9}
    assert (M.PLANE_DEMO_CLIP, M.PLANE_DEMO_TIME, M.PLANE_REPLAY_KEEP, M.PLANE_REPLAY_SUBSET, M.PLANE_RING_PERM) == (5, 6, 7, 8, 9)
    # the planes documented before them: e, e + 2^32, e + 2^33, e + 3 * 2^32, e + 4 * 2^32
    for row in ("index e            x:", "index e + 2^32", "index e + 2^33", "index e + 3 * 2^32", "index e + 4 * 2^32"):
        assert row in h
    assert not {0, 1, 2, 3, 4} & set(planes.values())
    for p in planes.values():
        assert re.search(rf"index (i|r) \+ {p} \* 2\^32|index {p} \* 2\^32", h), f"plane {p} missing from the draw table"


def test_new_structs_match_header():
    from pulse_b200 import _lib
    names = [("pulse_amp_ring_t", _lib.AmpRing), ("pulse_amp_demo_args_t", _lib.AmpDemoArgs), ("pulse_amp_store_args_t", _lib.AmpStoreArgs),
             ("pulse_amp_sample_args_t", _lib.AmpSampleArgs), ("pulse_ztask_reset_args_t", _lib.ZTaskResetArgs),
             ("pulse_amp_row_args_t", _lib.AmpRowArgs)]
    fmt = " ".join(["%zu"] * len(names))
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "pulse_b200.h"\nint main(){printf("' + fmt + ' %zu %zu\\n", '
           + ", ".join(f"sizeof({n})" for n, _ in names)
           + ', offsetof(pulse_ztask_reset_args_t, amp_fresh), offsetof(pulse_amp_row_args_t, amp_width));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        out = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert out == [C.sizeof(t) for _, t in names] + [_lib.ZTaskResetArgs.amp_fresh.offset, _lib.AmpRowArgs.amp_width.offset]
