"""The PULSE-X speed task (52-body SMPL-X humanoid) without a GPU: the oracle's restatement against the fixture written by the
UNMODIFIED reference (tests/golden/make_golden_smplx_speed.py), the pinned difference between the self observation's heading and the
task observation's, the C layout of the new argument structs, and the host-side refusals."""
import ctypes as C
import importlib.util
import os
import subprocess
import tempfile
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import pulse_oracle as po
from tests import smplx_speed_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def gen():
    spec = importlib.util.spec_from_file_location("make_golden_smplx_speed", os.path.join(HERE, "golden", "make_golden_smplx_speed.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_oracle_matches_reference_fixture():
    m = gen()
    g = np.load(os.path.join(HERE, "golden", "smplx_speed.npz"))
    z = m.inputs(int(g["num_envs"]))
    T = lambda k: torch.from_numpy(g[k])
    obs, rew, rs, tm = so.step(z, m.CONTACT_IDS, m.MAX_LEN, m.DT)
    close = lambda a, name: torch.testing.assert_close(a, T(name), atol=2e-6, rtol=2e-6, msg=lambda s: f"{name}: {s}")
    close(obs[:, :so.SELF_OBS], "self_obs")
    close(obs[:, so.SELF_OBS:], "speed_obs")
    close(rew, "speed_reward")
    close(po.remove_base_rot(z["body_state"][:, 0, 3:7]), "base_removed")
    assert torch.equal(rs, T("reset")) and torch.equal(tm, T("terminate"))
    _, _, rs_hi, tm_hi = so.step(z, m.CONTACT_IDS_HI, m.MAX_LEN, m.DT)
    assert torch.equal(rs_hi, T("reset_hi")) and torch.equal(tm_hi, T("terminate_hi"))
    pinned = torch.arange(2, z["progress_buf"].shape[0], 17)
    pinned = pinned[z["progress_buf"][pinned] > 1]
    assert pinned.numel() > 0 and bool(tm[pinned].all()) and not bool(tm_hi[pinned].any())   # body 40's contact bit decides
    assert int(tm.sum()) > 0 and int((z["progress_buf"] <= 1).sum()) > 0 and int((z["progress_buf"] >= m.MAX_LEN - 1).sum()) > 0


def reset_draws(g, n):
    """The reference reset's recorded draws (clips, start phases, task uniforms, change steps) per ENV, and the reset env ids."""
    ids = torch.from_numpy(g["r_env_ids"])
    d = {"motion_ids": torch.zeros(n, dtype=torch.int64), "phase": torch.zeros(n), "task_u": torch.zeros(n), "steps": torch.zeros(n, dtype=torch.int64)}
    assert str(g["r_draws"]) == "multinomial rand rand randint"
    for i, k in enumerate(("motion_ids", "phase", "task_u", "steps")):
        d[k][ids] = torch.from_numpy(g[f"r_draw{i}"])
    return ids, d


def reset_tables(m):
    from tests import ztask_reset_oracle as zo
    tb = so.tables(m.RESET_CLIPS, seed=m.TABLE_SEED)
    return tb, so.ground_table(tb, zo.StandInParser(), torch.linspace(-1.0, 1.0, 10))


def test_reset_oracle_matches_reference_fixture():
    """HumanoidSpeed's reset methods on a 52-body MotionLib (has_upright_start False): the oracle's sample_ref_state with the face-x
    adjustment and the ground fix from the per-frame floor table, and _reset_task, replayed on the recorded draws."""
    from tests import ztask_reset_oracle as zo
    m = gen()
    g = np.load(os.path.join(HERE, "golden", "smplx_speed.npz"))
    n = m.RESET_N
    ids, d = reset_draws(g, n)
    tb, floor = reset_tables(m)
    s = zo.sample_ref_state(tb, d["motion_ids"][ids], d["phase"][ids], floor, zo.FACE_X, False, zo.RANDOM)
    T = lambda k: torch.from_numpy(g[k])[ids]
    assert torch.equal(T("r_motion_ids"), d["motion_ids"][ids]) and torch.equal(T("r_start_times"), s["t0"])
    close = lambda a, k: torch.testing.assert_close(a, T(k), atol=1e-5, rtol=0, msg=lambda x: f"{k}: {x}")
    close(torch.cat([s["root_pos"], s["root_rot"], s["root_vel"], s["root_ang_vel"]], -1), "r_root_states")
    close(torch.cat([s["rb_pos"], s["rb_rot"], s["body_vel"], s["body_ang_vel"]], -1), "r_body_state")
    close(s["dof_pos"], "r_dof_pos")
    close(s["dof_vel"], "r_dof_vel")
    want, chg = zo.speed_task(d["task_u"][ids], d["steps"][ids], torch.from_numpy(g["r_progress"])[ids], **zo.SPEED)
    assert torch.equal(T("r_tar_speed"), want) and torch.equal(T("r_change_steps"), chg)


def test_self_and_task_headings_differ():
    """The self observation takes the heading of remove_base_rot(root), the task observation the raw root's: with rotations far from
    upright, the upright branch misses the fixture's self observation and a base-removed task heading misses its task observation."""
    m = gen()
    g = np.load(os.path.join(HERE, "golden", "smplx_speed.npz"))
    z = m.inputs(int(g["num_envs"]))
    upright = so.self_obs(z["body_state"], upright=True)
    assert float((upright - torch.from_numpy(g["self_obs"])).abs().amax(dim=1).min()) > 1e-3
    root = z["body_state"][:, 0].clone()
    root[:, 3:7] = po.remove_base_rot(root[:, 3:7])
    assert float((po.speed_obs(root, z["tar_speed"]) - torch.from_numpy(g["speed_obs"])).abs().amax(dim=1).min()) > 1e-3


def test_struct_sizes_match_header():
    from pulse_b200 import _lib
    src = ('#include <stdio.h>\n#include "pulse_b200.h"\nint main(){printf("%zu %zu %zu\\n", sizeof(pulse_smplx_motionlib_desc_t), '
           'sizeof(pulse_smplx_motion_query_t), sizeof(pulse_smplx_speed_step_args_t));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [C.sizeof(_lib.SmplxMotionLibDesc), C.sizeof(_lib.SmplxMotionQuery), C.sizeof(_lib.SmplxSpeedStepArgs)]


def test_entry_points_validate_arguments_without_gpu():
    from pulse_b200 import _lib
    from pulse_b200 import build
    build.build()
    lib = _lib.load()
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    a = _lib.SmplxSpeedStepArgs(body_state=ptr, obs_buf=ptr, tar_speed=ptr, body_env_stride=24 * 13, obs_stride=781)
    assert lib.pulse_smplx_speed_step(C.byref(a), 4, None) == -1 and b"body_env_stride" in lib.pulse_last_error()
    a.body_env_stride, a.obs_stride = 52 * 13, 361
    assert lib.pulse_smplx_speed_obs_list(C.byref(a), ptr, ptr, 4, None) == -1 and b"obs_stride" in lib.pulse_last_error()
    a.obs_stride = 781
    assert lib.pulse_smplx_speed_rollout_step(C.byref(a), ptr, 4, None) == -1 and b"null buffer" in lib.pulse_last_error()
    r = _lib.ZTaskResetArgs(reset_buf=ptr, env_list=ptr, count=ptr, sampled_motion_ids=ptr, motion_start_times=ptr, progress_buf=ptr,
                            root_states=ptr, dof_pos=ptr, dof_vel=ptr, rigid_body_state=ptr, root_env_stride=13, dof_elem_stride=1,
                            dof_env_stride=153, body_env_stride=52 * 13, amp_obs_buf=ptr, pose_mode=_lib.ZPOSE_FACE_X)
    h = C.c_void_p(C.addressof(buf))
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"AMP" in lib.pulse_last_error()
    r.amp_obs_buf, r.dof_env_stride = None, 69
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"strides" in lib.pulse_last_error()
    r.dof_env_stride, r.target_states = 153, ptr
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"target_states" in lib.pulse_last_error()
    r.target_states, r.pose_mode = None, _lib.ZPOSE_ROOT_XY_ZERO
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"pose_mode" in lib.pulse_last_error()
    d = _lib.SmplxMotionLibDesc()
    assert lib.pulse_smplx_motionlib_create(C.byref(d), None, C.byref(C.c_void_p())) == -1 and b"null table" in lib.pulse_last_error()


def _pieces(task_w=781, policy_w=781, S=778, A=153, E=48, reset_smplx=True, layout="smplx"):
    from pulse_b200 import _lib
    task = NS(kind=_lib.ZTASK_SPEED, obs_size=task_w, num_envs=4, layout=layout)
    reset = NS(kind="speed", smplx=reset_smplx, bodies=52 if reset_smplx else 24)
    policy = NS(obs_size=policy_w, A=E, disc=None, device="cpu")
    return task, reset, policy, NS(E=E, S=S, A=A)


def test_driver_accepts_smplx_pieces_and_rejects_mismatches():
    from pulse_b200 import PulseError, ZTaskStepsB200
    from pulse_b200.ztask_rollout import check_pieces
    assert check_pieces(*_pieces()) == "speed"
    bad = [_pieces(task_w=361, policy_w=361),          # the SMPL observation width
           _pieces(policy_w=780),                      # policy and step disagree
           _pieces(S=358),                             # an SMPL decoder
           _pieces(A=69),
           _pieces(E=32),                              # the PULSE-X latent is 48-dimensional
           _pieces(reset_smplx=False),                 # an SMPL reset
           _pieces(layout="smpl")]                     # an SMPL-X reset under an SMPL step
    for pieces in bad:
        with pytest.raises(PulseError):
            ZTaskStepsB200(*pieces, sim={})
    t, r, p, v = _pieces()
    sim = {k: None for k in ("body_state", "root_states", "dof_pos", "dof_vel", "progress_buf", "sampled_motion_ids", "motion_start_times")}
    with pytest.raises(PulseError, match="dof_force"):
        ZTaskStepsB200(t, r, p, v, sim=dict(sim, dof_force=torch.zeros(4, 153)))


def test_step_object_rejects_power_terms_and_bad_bodies():
    from pulse_b200 import PulseError
    from pulse_b200.ztasks import SmplxSpeedTaskB200
    with pytest.raises(PulseError, match="power"):
        SmplxSpeedTaskB200(4, "cpu", contact_body_ids=(7, 3, 8, 4), power_reward=True)
    with pytest.raises(PulseError, match="contact_body_ids"):
        SmplxSpeedTaskB200(4, "cpu", contact_body_ids=(7, 52))


def test_smplx_tables_never_reach_an_smpl_entry_point():
    """A 52-body MotionLibB200 refuses its SMPL handle, so the SMPL consumers (HumanoidImCompute, the SMPL resets) raise PulseError instead
    of reading the SMPL-X handle as an SMPL one; a 24-body one refuses the SMPL-X handle."""
    from pulse_b200 import PulseError
    from pulse_b200.humanoid_im import HumanoidImCompute
    from pulse_b200.motion_lib import MotionLibB200
    libs = {}
    for smplx in (True, False):
        ml = MotionLibB200.__new__(MotionLibB200)           # no device here: the attributes a built one has
        ml.smplx, ml._handle, ml._device = smplx, C.c_void_p(0), torch.device("cpu")
        libs[smplx] = ml
    with pytest.raises(PulseError, match="SMPL-X"):
        libs[True].handle
    with pytest.raises(PulseError, match="SMPL-X"):
        HumanoidImCompute(libs[True])
    with pytest.raises(PulseError, match="no SMPL-X handle"):
        libs[False].smplx_handle
    assert libs[True].smplx_handle is libs[True]._handle and libs[False].handle is libs[False]._handle
