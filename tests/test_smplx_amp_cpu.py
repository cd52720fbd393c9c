"""The PULSE-X AMP rows (52-body SMPL-X humanoid, env_pulsex_amp.yaml) without a GPU: the float64 restatement (tests/smplx_amp_fp64.py)
against the fixture written by the UNMODIFIED reference (tests/golden/make_golden_smplx_amp.py), the width arithmetic, the host-side
refusals and the entry points' argument checks."""
import ctypes as C
import importlib.util
import os
import re
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests import reset_fp64 as rf
from tests import smplx_amp_fp64 as xf
from tests import smplx_speed_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def gen():
    spec = importlib.util.spec_from_file_location("make_golden_smplx_amp", os.path.join(HERE, "golden", "make_golden_smplx_amp.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def golden():
    return np.load(os.path.join(HERE, "golden", "smplx_amp.npz"))


def golden_rows(g, key: str, width: int) -> np.ndarray:
    """The fixture's 466-float rows `key` at `width`: 465 drops the root height, the first column (the generator checks that the
    reference's 465-float rows are exactly these)."""
    rows = g[key]
    return rows if width == xf.AMP_OBS else rows[..., 1:]


def close(got, want, what):
    torch.testing.assert_close(got, torch.from_numpy(np.ascontiguousarray(want)).double(), atol=2e-5, rtol=2e-5, msg=lambda s: f"{what}: {s}")


def test_width_arithmetic():
    from pulse_b200 import _lib
    assert xf.J == 49 and len(xf.DOF_SUBSET) == 147
    assert xf.AMP_OBS == 1 + 6 + 3 + 3 + 49 * 6 + 49 * 3 + 4 * 3 == 466 and xf.AMP_OBS_NO_HEIGHT == 465
    assert 10 * xf.AMP_OBS_NO_HEIGHT == 4650 and 10 * xf.AMP_OBS_NO_HEIGHT * 4 == 18600
    assert (_lib.SMPLX_AMP_OBS, _lib.SMPLX_AMP_OBS_NO_HEIGHT) == (466, 465)
    hdr = open(os.path.join(ROOT, "include", "pulse_b200.h")).read()
    assert int(re.search(r"#define PULSE_SMPLX_AMP_OBS (\d+)", hdr).group(1)) == 466
    assert int(re.search(r"#define PULSE_SMPLX_AMP_OBS_NO_HEIGHT (\d+)", hdr).group(1)) == 465
    from pulse_b200.ztask_reset import SMPLX_DOF_SUBSET, SMPLX_KEY_BODY_IDS
    g = golden()
    assert list(SMPLX_DOF_SUBSET) == xf.DOF_SUBSET == g["dof_subset"].tolist()
    assert list(SMPLX_KEY_BODY_IDS) == xf.KEY_BODIES == g["key_body_ids"].tolist()


@pytest.mark.parametrize("height", [True, False])
def test_state_rows_match_reference_fixture(height):
    """build_amp_observations_smpl of the reference on seeded 52-body states, far from upright, against the float64 restatement."""
    m, g = gen(), golden()
    bs, dof_pos, dof_vel = m.state_inputs()
    ref = xf.state_amp_ref(bs, dof_pos, dof_vel, upright=False)
    width = 466 if height else 465
    assert not bool(ref["ill"].any())
    want = golden_rows(g, "state_amp", width)
    close(xf.ref_values(ref, width), want, f"state rows, width {width}")
    # the kernel's bounds hold the reference's fp32 rows too
    xf.check_amp(None, f"fixture state rows {width}", torch.from_numpy(np.ascontiguousarray(want)), ref)
    # the upright heading misses them: remove_base_rot is applied
    up = xf.ref_values(xf.state_amp_ref(bs, dof_pos, dof_vel, upright=True), width)
    assert float((up - torch.from_numpy(np.ascontiguousarray(want)).double()).abs().amax(1).min()) > 1e-3


def test_dropped_toe_dofs_are_nonzero_and_absent():
    """The fixture's toe dofs are non-zero, and no column of its rows equals them: they never leak into the row."""
    m, g = gen(), golden()
    _, dof_pos, dof_vel = m.state_inputs()
    toes = [3 * j + c for j in (3, 7) for c in range(3)]
    assert bool((dof_vel[:, toes] != 0).all()) and bool((dof_pos[:, toes] != 0).all())
    row = torch.from_numpy(g["state_amp"])
    for c in toes:
        assert not bool((row == dof_vel[:, c:c + 1]).all(0).any()), f"dof {c}'s velocity is a column of the rows"


@pytest.mark.parametrize("height", [True, False])
def test_motion_rows_match_reference_fixture(height):
    """_init_amp_obs_ref (t0 - k dt, k >= 1) and build_amp_obs_demo_steps (k >= 0) on the 52-body stand-in, against the float64 motion
    row at the same times."""
    m, g = gen(), golden()
    tb, mids, t0 = m.ref_inputs()
    assert torch.equal(mids, torch.from_numpy(g["ref_motion_ids"])) and torch.equal(t0, torch.from_numpy(g["ref_t0"]))
    td = so.table_dict(tb)
    width = 466 if height else 465
    times = rf.history_times(t0, m.DT, m.STEPS)
    init, demo = golden_rows(g, "init", width), golden_rows(g, "demo", width)
    for k in range(m.STEPS):
        ref = xf.motion_amp_ref(rf.motion_ref(td, mids, times[:, k]))
        if k >= 1:
            close(xf.ref_values(ref, width), init[:, k - 1], f"_init_amp_obs_ref row {k}, width {width}")
        close(xf.ref_values(ref, width), demo[:, k], f"build_amp_obs_demo_steps row {k}, width {width}")


def test_host_refusals():
    from pulse_b200 import PulseError
    from pulse_b200.amp_buffers import AmpBuffersB200
    from pulse_b200.ztask_reset import check_amp_layout
    smplx, smpl = NS(smplx=True, _device=torch.device("cpu")), NS(smplx=False, _device=torch.device("cpu"))
    for ml, width, upright, what in ((smplx, 196, False, "465"), (smplx, 195, False, "465"), (smpl, 465, True, "195"), (smpl, 466, False, "195"),
                                     (smplx, 465, True, "upright=False")):
        with pytest.raises(PulseError, match=what):
            AmpBuffersB200(ml, amp_width=width, upright=upright)
    m = gen()
    task = lambda **k: NS(**dict(dict(amp_obs_v=1, _key_body_ids=torch.tensor(m.KEY_BODY_IDS), dof_subset=torch.tensor(m.DOF_SUBSET),
                                      _has_dof_subset=True), **k))
    check_amp_layout(task(), "t", smplx=True)
    for bad, what in ((task(_key_body_ids=torch.tensor([7, 3, 22, 17])), "keyBodies"), (task(_key_body_ids=torch.tensor([7, 3, 37, 17])), "keyBodies"),
                      (task(dof_subset=torch.tensor([k for k in range(153) if k // 3 not in (3, 7, 17)])), "dof_subset"),
                      (task(_has_dof_subset=False), "dof_subset"), (task(amp_obs_v=2), "amp_obs_v")):
        with pytest.raises(PulseError, match=what):
            check_amp_layout(bad, "t", smplx=True)
    with pytest.raises(PulseError, match="keyBodies"):                 # an SMPL-X task is not an SMPL one
        check_amp_layout(task(), "t")


def _pieces(amp_width=465, reset_width=465, upright=False, disc=4650):
    from pulse_b200 import _lib
    task = NS(kind=_lib.ZTASK_SPEED, obs_size=781, num_envs=4, layout="smplx")
    reset = NS(kind="speed", smplx=True, bodies=52, amp_width=reset_width, upright=False)
    policy = NS(obs_size=781, A=48, disc=NS(size=disc), device="cpu")
    amp = NS(amp_width=amp_width, upright=upright, num_steps=10, row_floats=10 * amp_width, layout="smplx")
    return task, reset, policy, NS(E=48, S=778, A=153), amp


def test_driver_accepts_the_smplx_amp_part():
    from pulse_b200 import PulseError
    from pulse_b200.ztask_rollout import check_pieces
    assert check_pieces(*_pieces()) == "speed"
    for pieces in (_pieces(amp_width=466), _pieces(amp_width=195), _pieces(upright=True)):
        with pytest.raises(PulseError, match="AMP part"):
            check_pieces(*pieces)


def test_entry_points_validate_arguments_without_gpu():
    from pulse_b200 import _lib
    from pulse_b200 import build
    build.build()
    lib = _lib.load()
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    p2 = C.cast(C.addressof(buf) + 4 * 32, C.c_void_p)
    a = _lib.AmpRowArgs(body_state=ptr, body_env_stride=52 * 13, dof_pos=ptr, dof_vel=ptr, dof_env_stride=153, dof_elem_stride=1, prev=ptr,
                        ld_prev=9 * 465, out=p2, ld_out=10 * 465, num_steps=10, amp_width=465, remove_base_rot=1)
    for field, value, what in (("amp_width", 196, b"amp_width"), ("amp_width", 0, b"amp_width"), ("remove_base_rot", 0, b"remove_base_rot"),
                               ("body_env_stride", 24 * 13, b"body_env_stride"), ("dof_env_stride", 69, b"dof strides"),
                               ("ld_out", 10 * 465 - 1, b"strides"), ("num_steps", 17, b"num_steps")):
        bad = _lib.AmpRowArgs.from_buffer_copy(a)
        setattr(bad, field, value)
        assert lib.pulse_smplx_amp_obs_row(C.byref(bad), 4, None) == -1 and what in lib.pulse_last_error(), field
    s = _lib.AmpRowArgs.from_buffer_copy(a)
    s.ld_prev, s.ld_out = 9 * 465, 10 * 465
    assert lib.pulse_amp_obs_row(C.byref(s), 4, None) == -1 and b"amp_width" in lib.pulse_last_error()   # SMPL-X rows, SMPL entry point
    ring = _lib.AmpRing(rows=ptr, capacity=8, ctr=ptr, seed=1, row_floats=10 * 465)
    d = _lib.AmpDemoArgs(ring=ring, sampling_cdf=ptr, num_samples=4, num_steps=10, amp_width=465, upright=0, dt=0.033)
    smpl_desc, smplx_desc = _lib.MotionLibDesc(num_motions=1, aux_rec=ptr), _lib.SmplxMotionLibDesc(num_motions=1, aux_rec=ptr)
    smpl_h, smplx_h = C.c_void_p(C.addressof(smpl_desc)), C.c_void_p(C.addressof(smplx_desc))   # a handle holds its descriptor
    assert lib.pulse_amp_demo_fetch(smpl_h, C.byref(d), None) == -1 and b"amp_width 465" in lib.pulse_last_error()
    d.amp_width, d.ring.row_floats = 196, 1960
    assert lib.pulse_smplx_amp_demo_fetch(smplx_h, C.byref(d), None) == -1 and b"amp_width 196" in lib.pulse_last_error()
    d.amp_width, d.ring.row_floats, d.upright = 465, 4650, 1
    assert lib.pulse_smplx_amp_demo_fetch(smplx_h, C.byref(d), None) == -1 and b"upright" in lib.pulse_last_error()
    h = C.c_void_p(C.addressof(buf))
    r = _lib.ZTaskResetArgs(reset_buf=ptr, env_list=ptr, count=ptr, sampled_motion_ids=ptr, motion_start_times=ptr, progress_buf=ptr,
                            root_states=ptr, dof_pos=ptr, dof_vel=ptr, rigid_body_state=ptr, root_env_stride=13, dof_elem_stride=1,
                            dof_env_stride=153, body_env_stride=52 * 13, amp_obs_buf=ptr, num_amp_steps=10, amp_width=195,
                            pose_mode=_lib.ZPOSE_FACE_X)
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"amp_width 195" in lib.pulse_last_error()
    r.amp_width, r.num_amp_steps = 465, 17
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"num_amp_steps" in lib.pulse_last_error()
    r.amp_obs_buf, r.amp_fresh = None, ptr
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"amp_fresh" in lib.pulse_last_error()
