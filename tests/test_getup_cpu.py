"""CPU checks of the getup reset: the oracle (tests/getup_oracle.py) against the unmodified reference's `_reset_actors` rounds recorded in
tests/golden/getup.npz, the conversion of the reference's draws into the kernel's injected form, the C ABI of `pulse_reset_getup` /
`pulse_getup_amp_init`, and the attribute contract of `HumanoidImGetupB200Mixin`."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import getup_oracle as go
from tests.helpers import load_npz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx():
    return load_npz("getup.npz")


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def _rounds(fx, case):
    n = int(fx[f"{case}_n"])
    st = {"avail": fx[f"{case}_init_avail"], "fid": fx[f"{case}_init_fid"], "recovery_counter": fx[f"{case}_init_rc"],
          "root_states": fx[f"{case}_init_root"], "dof_pos": fx[f"{case}_init_dof_pos"], "dof_vel": fx[f"{case}_init_dof_vel"],
          "fall_root": fx[f"{case}_init_fall_root"], "fall_dof_pos": fx[f"{case}_init_fall_dof_pos"],
          "fall_dof_vel": fx[f"{case}_init_fall_dof_vel"]}
    for r in range(int(fx[f"{case}_rounds"])):
        p = f"{case}_r{r}_"
        yield n, st, {k[len(p):]: v for k, v in fx.items() if k.startswith(p)}


@pytest.mark.parametrize("case", ["a", "b"])
def test_oracle_reproduces_reference_rounds(fx, case):
    """Masks, assignments, availability, counters and written states of every round, bit for bit; the stale release (case a) and the
    exhausted pool (case b) included."""
    p_rec, p_fall, steps = float(fx[f"{case}_p_rec"]), float(fx[f"{case}_p_fall"]), int(fx[f"{case}_steps"])
    for n, st, r in _rounds(fx, case):
        st["terminate_buf"] = r["terminate"]
        perm = r["perm"] if r["perm"].numel() else None
        draws = go.draws_from_reference(r["env_ids"], r["terminate"], st["avail"], st["fid"], r["rec_bern"], r["fall_bern"], perm, n)
        o, info = go.getup_reset_actors(st, r["env_ids"], *draws, p_rec, p_fall, steps)
        if int(r["assert"]):
            # the reference asserts: the oracle (and the kernel) give the surplus a reference-state episode instead
            rec = info["recovery_ids"]
            assert info["shortfall"] > 0 and torch.equal(o["recovery_counter"][rec], r["rc"][rec])
            return
        assert info["shortfall"] == 0
        assert torch.equal(info["ref_ids"], r["ref_ids"])
        for k, ref in (("avail", "avail"), ("fid", "fid"), ("recovery_counter", "rc"), ("root_states", "root"), ("dof_pos", "dof_pos"),
                       ("dof_vel", "dof_vel")):
            assert torch.equal(o[k], r[ref]), k
        st.update({k: o[k] for k in ("avail", "fid", "recovery_counter", "root_states", "dof_pos", "dof_vel")})   # the next round's state
    assert case == "a" and int(fx["a_stale_releases"]) > 0


def test_draw_conversion_is_exact(fx):
    """The injected uniforms reproduce each recorded Bernoulli result, and the keys order the free states exactly as the permutation."""
    for case in ("a", "b"):
        p_rec, p_fall = float(fx[f"{case}_p_rec"]), float(fx[f"{case}_p_fall"])
        for n, st, r in _rounds(fx, case):
            ids = r["env_ids"]
            perm = r["perm"] if r["perm"].numel() else None
            rec_u, fall_u, keys = go.draws_from_reference(ids, r["terminate"], st["avail"], st["fid"], r["rec_bern"], r["fall_bern"], perm, n)
            assert torch.equal((rec_u[ids] < p_rec).float(), r["rec_bern"])
            non = ids[~((r["rec_bern"] == 1) & (r["terminate"][ids] == 1))]
            assert torch.equal((fall_u[non] < p_fall).float(), r["fall_bern"])
            if perm is not None:
                a = st["avail"].clone()
                a[st["fid"][ids]] = 0
                free = a.eq(0).nonzero().flatten()
                assert torch.equal(free[torch.argsort(keys[free], stable=True)], free[perm])
            st.update(avail=r["avail"], fid=r["fid"])
    # the edge probabilities: a success is only ever recorded for p > 0, a failure for p < 1
    for p, b in ((0.0, 0.0), (1.0, 1.0), (0.3, 1.0), (0.3, 0.0)):
        rec_u, _, _ = go.draws_from_reference(torch.tensor([0]), torch.ones(1, dtype=torch.long), torch.zeros(1, dtype=torch.long),
                                              torch.zeros(1, dtype=torch.long), torch.tensor([b]), torch.zeros(1 - int(b)), None, 1)
        assert float(rec_u[0] < p) == b


def test_getup_symbols_and_struct_layout(lib):
    import subprocess
    import tempfile
    from pulse_b200 import _lib
    for n in ("pulse_reset_getup", "pulse_getup_amp_init"):
        assert hasattr(lib, n) and n in _lib.SIGNATURES
    assert lib.pulse_abi_version() == 3
    fields = ("recovery_u", "recovery_prob", "recovery_steps", "recovery_counter", "fall_root_stride", "num_fall_states", "class_counts",
              "env_class", "error", "fall_key_scratch")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "pulse_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu", sizeof(pulse_getup_reset_args_t), '
           'sizeof(pulse_getup_amp_args_t), sizeof(pulse_reset_args_t), offsetof(pulse_getup_amp_args_t, class_counts), '
           'offsetof(pulse_getup_amp_args_t, num_steps));'
           + "".join(f'printf(" %zu", offsetof(pulse_getup_reset_args_t, {f}));' for f in fields) + 'return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert got == [C.sizeof(_lib.GetupResetArgs), C.sizeof(_lib.GetupAmpArgs), C.sizeof(_lib.ResetArgs), _lib.GetupAmpArgs.class_counts.offset,
                   _lib.GetupAmpArgs.num_steps.offset] + [getattr(_lib.GetupResetArgs, f).offset for f in fields]
    assert (_lib.GETUP_REF, _lib.GETUP_FALL, _lib.GETUP_RECOVERY) == (go.REF, go.FALL, go.RECOVERY)


def test_getup_entry_points_validate_arguments_without_gpu(lib):
    from pulse_b200 import _lib
    assert lib.pulse_reset_getup(None, None, 4, None) == -1 and b"null" in lib.pulse_last_error()
    assert lib.pulse_getup_amp_init(None, 4, None) == -1 and b"null" in lib.pulse_last_error()
    buf = (C.c_float * 256)()
    ptr = C.cast(buf, C.c_void_p)
    desc = _lib.MotionLibDesc(aux_rec=ptr)              # a handle is its descriptor (pulse_common.cuh)
    fake_lib = C.cast(C.pointer(desc), C.c_void_p)
    g = _lib.GetupResetArgs()
    assert lib.pulse_reset_getup(fake_lib, C.byref(g), 4, None) == -1 and b"mask" in lib.pulse_last_error()
    b = g.base
    b.reset_buf = b.env_list = b.count = ptr
    b.motion_ids = b.motion_start_times = b.motion_start_offset = b.global_offset = b.progress_buf = ptr
    b.root_states = b.dof_pos = b.dof_vel = ptr
    b.root_env_stride, b.dof_env_stride, b.dof_elem_stride = 13, 138, 2
    g.base = b
    assert lib.pulse_reset_getup(fake_lib, C.byref(g), 4, None) == -1 and b"terminate_buf" in lib.pulse_last_error()
    g.base.terminate_buf = ptr
    assert lib.pulse_reset_getup(fake_lib, C.byref(g), 4, None) == -1 and b"getup buffer" in lib.pulse_last_error()
    g.recovery_counter = g.available_fall_states = g.fall_id_assignments = ptr
    g.ref_list = g.fall_list = g.recovery_list = g.class_counts = g.error = g.fall_pick = g.fall_key_scratch = ptr
    assert lib.pulse_reset_getup(fake_lib, C.byref(g), 4, None) == -1 and b"num_fall_states" in lib.pulse_last_error()
    g.num_fall_states = 4
    g.fall_root_states = g.fall_dof_pos = g.fall_dof_vel = ptr
    g.fall_root_stride, g.fall_dof_env_stride, g.fall_dof_elem_stride = 13, 60, 1
    assert lib.pulse_reset_getup(fake_lib, C.byref(g), 4, None) == -1 and b"fall-state strides" in lib.pulse_last_error()
    a = _lib.GetupAmpArgs(body_state=ptr, dof_pos=ptr, dof_vel=ptr, amp_obs_buf=ptr, fall_list=ptr, recovery_list=ptr, class_counts=ptr,
                          num_steps=20, body_env_stride=312)
    assert lib.pulse_getup_amp_init(C.byref(a), 4, None) == -1 and b"num_steps" in lib.pulse_last_error()


def test_getup_mixin_reads_only_reference_names(fx):
    """Every attribute HumanoidImGetupB200Mixin reads from `self` is the base mixin's contract, a name the reference's
    humanoid_im_getup.py uses (recorded in the fixture), defined by the mixins, or private to them (`_pulse*`)."""
    import ast
    from tests.standins import CONTRACT
    tree = ast.parse(open(os.path.join(ROOT, "pulse_b200", "humanoid_im.py")).read())
    classes = {n.name: n for n in ast.walk(tree) if isinstance(n, ast.ClassDef)}
    defined = {f.name for c in ("HumanoidImB200Mixin", "HumanoidImGetupB200Mixin") for f in classes[c].body if isinstance(f, ast.FunctionDef)}
    reads = set()
    for node in ast.walk(classes["HumanoidImGetupB200Mixin"]):
        if isinstance(node, ast.Attribute) and isinstance(node.value, ast.Name) and node.value.id == "self":
            reads.add(node.attr)
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "getattr" and len(node.args) >= 2 \
                and isinstance(node.args[0], ast.Name) and node.args[0].id == "self" and isinstance(node.args[1], ast.Constant):
            reads.add(node.args[1].value)
    allowed = set(n for names in CONTRACT["task"].values() for n in names) | set(fx["names"].split()) | defined
    unknown = sorted(a for a in reads if a not in allowed and a not in ("device", "num_envs") and not a.startswith("_pulse"))
    assert not unknown, unknown
