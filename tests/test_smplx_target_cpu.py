"""The PULSE-X reach and strike tasks (52-body SMPL-X humanoid) without a GPU: the oracle restatement against the fixture written by the
UNMODIFIED reference (tests/golden/make_golden_smplx_target.py), the reset oracle replaying the reference's recorded draws, the C
layout of the step argument struct, the entry points' argument checks, and the host-side refusals."""
import ctypes as C
import importlib.util
import os
import subprocess
import tempfile
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests import smplx_speed_oracle as so
from tests import smplx_target_oracle as to

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIXTURE = os.path.join(HERE, "golden", "smplx_target.npz")


def gen():
    spec = importlib.util.spec_from_file_location("make_golden_smplx_target", os.path.join(HERE, "golden", "make_golden_smplx_target.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_oracle_matches_reference_fixture():
    m, sm = gen(), gen().speed_gen()
    g = np.load(FIXTURE)
    z = m.inputs(int(g["num_envs"]))
    T = lambda k: torch.from_numpy(g[k])
    close = lambda a, name: torch.testing.assert_close(a, T(name), atol=2e-6, rtol=2e-6, msg=lambda s: f"{name}: {s}")
    for tag, ids in (("", sm.CONTACT_IDS), ("_hi", sm.CONTACT_IDS_HI)):
        for b in m.REACH_IDS:
            obs, rew, rs, tm = to.step(z, "reach", ids, sm.MAX_LEN, sm.DT, reach_id=b)
            close(obs[:, :so.SELF_OBS], "self_obs")
            close(obs[:, so.SELF_OBS:], "reach_obs")
            close(rew, f"reach_reward_{b}")
            assert torch.equal(rs, T("reach_reset" + tag)) and torch.equal(tm, T("reach_terminate" + tag))
        obs, rew, rs, tm = to.step(z, "strike", ids, sm.MAX_LEN, sm.DT, strike_ids=m.STRIKE_IDS)
        close(obs[:, :so.SELF_OBS], "self_obs")
        close(obs[:, so.SELF_OBS:], "strike_obs")
        close(rew, "strike_reward")
        assert torch.equal(rs, T("strike_reset" + tag)) and torch.equal(tm, T("strike_terminate" + tag))
    prog = z["progress_buf"]
    pushed, strike_only = torch.arange(4, len(prog), 13), torch.arange(6, len(prog), 13)
    pushed, strike_only = pushed[prog[pushed] > 1], strike_only[prog[strike_only] > 1]
    tm = T("strike_terminate")
    assert pushed.numel() and bool(tm[pushed].all()) and not bool(T("reach_terminate")[pushed].any())   # only the pushed target fails them
    assert strike_only.numel() and not bool(tm[strike_only].any())        # body 45 is a strike body: the 64-bit strike mask
    assert bool((T("strike_reward")[8::13] == 1.0).all())                 # rot_err < 0.2
    ts, root = z["target_states"], z["body_state"][:, 0]
    d = torch.nn.functional.normalize(ts[10::13, 0:2] - root[10::13, 0:2], dim=-1)
    assert bool(((d * (root[10::13, 0:2] - z["prev_root_pos"][10::13, 0:2])).sum(-1) < 0).all())   # dir_speed <= 0 in those rows


def reset_draws(g, kind, n):
    """The reference reset's recorded draws per ENV and the reset env ids."""
    ids = torch.from_numpy(g[f"{kind}_r_env_ids"])
    p = f"{kind}_r_"
    if kind == "reach":
        assert str(g[p + "draws"]) == "multinomial rand rand randint"
        d = {"motion_ids": torch.zeros(n, dtype=torch.int64), "phase": torch.zeros(n), "task_u": torch.zeros(n, 3), "steps": torch.zeros(n, dtype=torch.int64)}
        for i, k in enumerate(("motion_ids", "phase", "task_u", "steps")):
            d[k][ids] = torch.from_numpy(g[p + f"draw{i}"])
    else:
        assert str(g[p + "draws"]) == "multinomial rand rand rand rand rand"
        d = {"motion_ids": torch.zeros(n, dtype=torch.int64), "phase": torch.zeros(n), "strike_u": torch.zeros(n, 4)}
        d["motion_ids"][ids], d["phase"][ids] = torch.from_numpy(g[p + "draw0"]), torch.from_numpy(g[p + "draw1"])
        for c in range(4):
            d["strike_u"][ids, c] = torch.from_numpy(g[p + f"draw{c + 2}"])
    return ids, d


@pytest.mark.parametrize("kind", ["reach", "strike"])
def test_reset_oracle_matches_reference_fixture(kind):
    """HumanoidReach / HumanoidStrike reset methods on a 52-body MotionLib: the oracle's sample_ref_state with the root's xy zeroed and
    the ground fix, the strike target and reach's _reset_task, replayed on the recorded draws."""
    from tests import ztask_reset_oracle as zo
    from tests.test_smplx_speed_cpu import reset_tables
    sm = gen().speed_gen()
    g = np.load(FIXTURE)
    ids, d = reset_draws(g, kind, sm.RESET_N)
    tb, floor = reset_tables(sm)
    s = zo.sample_ref_state(tb, d["motion_ids"][ids], d["phase"][ids], floor, zo.ROOT_XY_ZERO, False, zo.RANDOM)
    p = f"{kind}_r_"
    T = lambda k: torch.from_numpy(g[p + k])[ids]
    assert torch.equal(T("motion_ids"), d["motion_ids"][ids]) and torch.equal(T("start_times"), s["t0"])
    close = lambda a, want, k: torch.testing.assert_close(a, want, atol=1e-5, rtol=0, msg=lambda x: f"{k}: {x}")
    close(torch.cat([s["root_pos"], s["root_rot"], s["root_vel"], s["root_ang_vel"]], -1), T("root_states"), "root_states")
    assert bool((s["root_pos"][:, :2] == 0).all())
    close(torch.cat([s["rb_pos"], s["rb_rot"], s["body_vel"], s["body_ang_vel"]], -1), torch.from_numpy(g[p + "body_state"]), "body_state")
    close(s["dof_pos"], torch.from_numpy(g[p + "dof_pos"]), "dof_pos")
    close(s["dof_vel"], torch.from_numpy(g[p + "dof_vel"]), "dof_vel")
    if kind == "strike":
        close(zo.reset_target(s["root_pos"][:, :2], d["strike_u"][ids], **zo.STRIKE), T("target_states"), "target_states")
    else:
        want, chg = zo.reach_task(d["task_u"][ids], d["steps"][ids], torch.from_numpy(g[p + "progress"])[ids], **zo.REACH)
        close(want, T("tar_pos"), "tar_pos")
        assert torch.equal(T("change_steps"), chg)


def test_struct_size_matches_header():
    from pulse_b200 import _lib
    src = '#include <stdio.h>\n#include "pulse_b200.h"\nint main(){printf("%zu\\n", sizeof(pulse_smplx_target_step_args_t));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        size = int(subprocess.check_output([os.path.join(d, "s")]))
    assert size == C.sizeof(_lib.SmplxTargetStepArgs)


def test_entry_points_validate_arguments_without_gpu():
    from pulse_b200 import _lib
    from pulse_b200 import build
    build.build()
    lib = _lib.load()
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    err = lambda: lib.pulse_last_error()
    a = _lib.SmplxTargetStepArgs(kind=_lib.ZTASK_SPEED, body_state=ptr, obs_buf=ptr, tar_pos=ptr, body_env_stride=52 * 13, obs_stride=781,
                                 progress_buf=ptr, rew_buf=ptr, reset_buf=ptr, terminate_buf=ptr, termination_heights=ptr, reach_body_id=52)
    for fn in (lambda: lib.pulse_smplx_target_step(C.byref(a), 4, None), lambda: lib.pulse_smplx_target_obs_list(C.byref(a), ptr, ptr, 4, None),
               lambda: lib.pulse_smplx_target_rollout_step(C.byref(a), ptr, 4, None)):
        assert fn() == -1 and b"task kind" in err()
    a.kind = _lib.ZTASK_REACH
    assert lib.pulse_smplx_target_step(C.byref(a), 4, None) == -1 and b"reach_body_id" in err()
    a.reach_body_id, a.contact_body_mask = 51, 1 << 52
    assert lib.pulse_smplx_target_rollout_step(C.byref(a), ptr, 4, None) == -1 and b"mask" in err()
    a.contact_body_mask, a.strike_body_mask = 1 << 7, 1 << 63
    assert lib.pulse_smplx_target_step(C.byref(a), 4, None) == -1 and b"mask" in err()
    a.strike_body_mask, a.obs_stride = 1 << 45, 780
    assert lib.pulse_smplx_target_obs_list(C.byref(a), ptr, ptr, 4, None) == -1 and b"obs_stride" in err()
    a.kind, a.obs_stride, a.target_states, a.target_env_stride = _lib.ZTASK_STRIKE, 792, ptr, 13
    assert lib.pulse_smplx_target_step(C.byref(a), 4, None) == -1 and b"obs_stride" in err()
    a.obs_stride, a.target_states = 793, None
    assert lib.pulse_smplx_target_obs_list(C.byref(a), ptr, ptr, 4, None) == -1 and b"target_states" in err()
    a.target_states, a.prev_root_pos, a.dt = ptr, ptr, 1.0 / 30.0
    assert lib.pulse_smplx_target_step(C.byref(a), 4, None) == -1 and b"tar_contact_forces" in err()
    r = _lib.ZTaskResetArgs(reset_buf=ptr, env_list=ptr, count=ptr, sampled_motion_ids=ptr, motion_start_times=ptr, progress_buf=ptr,
                            root_states=ptr, dof_pos=ptr, dof_vel=ptr, rigid_body_state=ptr, root_env_stride=13, dof_elem_stride=1,
                            dof_env_stride=153, body_env_stride=52 * 13, pose_mode=_lib.ZPOSE_FACE_X)
    h = C.c_void_p(C.addressof(buf))
    assert lib.pulse_reset_smplx_target(h, C.byref(r), 4, None) == -1 and b"pose_mode" in err()
    r.pose_mode, r.dof_env_stride = _lib.ZPOSE_ROOT_XY_ZERO, 69
    assert lib.pulse_reset_smplx_target(h, C.byref(r), 4, None) == -1 and b"strides" in err()
    r.dof_env_stride, r.amp_obs_buf, r.amp_width, r.num_amp_steps = 153, ptr, 195, 10
    assert lib.pulse_reset_smplx_target(h, C.byref(r), 4, None) == -1 and b"amp_width" in err()
    # the speed task's SMPL-X reset keeps refusing the strike target and the reach / strike pose
    r.amp_obs_buf, r.target_states, r.target_env_stride = None, ptr, 13
    assert lib.pulse_reset_ztask_smplx(h, C.byref(r), 4, None) == -1 and b"target_states" in err()


def _pieces(kind="strike", task_w=793, policy_w=793, S=778, A=153, E=48, reset_smplx=True, layout="smplx", reset_kind=None):
    from pulse_b200 import _lib
    codes = {"reach": _lib.ZTASK_REACH, "speed": _lib.ZTASK_SPEED, "strike": _lib.ZTASK_STRIKE}
    task = NS(kind=codes[kind], obs_size=task_w, num_envs=4, layout=layout)
    reset = NS(kind=reset_kind or kind, smplx=reset_smplx, bodies=52 if reset_smplx else 24)
    policy = NS(obs_size=policy_w, A=E, disc=None, device="cpu")
    return task, reset, policy, NS(E=E, S=S, A=A)


def test_driver_accepts_smplx_target_pieces_and_rejects_mismatches():
    from pulse_b200 import PulseError, ZTaskStepsB200
    from pulse_b200.ztask_rollout import check_pieces
    assert check_pieces(*_pieces("strike")) == "strike"
    assert check_pieces(*_pieces("reach", 781, 781)) == "reach"
    bad = [_pieces("strike", layout="smpl", task_w=373, policy_w=373),   # an SMPL strike step with an SMPL-X reset
           _pieces("strike", policy_w=373),                              # a 373-wide policy under the SMPL-X strike step
           _pieces("strike", 373, 373),
           _pieces("reach", 793, 793),                                   # the strike width under reach
           _pieces("reach", 781, 781, reset_kind="speed"),               # a speed reset under a reach step
           _pieces("reach", 781, 781, reset_smplx=False),                # an SMPL reset
           _pieces("strike", S=358, A=69),                               # an SMPL decoder
           _pieces("reach", 781, 781, E=32)]                             # the PULSE-X latent is 48-dimensional
    for pieces in bad:
        with pytest.raises(PulseError):
            ZTaskStepsB200(*pieces, sim={})


def test_step_objects_refuse_what_they_do_not_serve():
    from pulse_b200 import PulseError
    from pulse_b200.ztasks import SmplxReachTaskB200, SmplxStrikeTaskB200
    feet = (7, 3, 8, 4)
    with pytest.raises(PulseError, match="reach_body_id"):
        SmplxReachTaskB200(4, "cpu", reach_body_id=52, contact_body_ids=feet)
    with pytest.raises(PulseError, match="contact_body_ids"):
        SmplxReachTaskB200(4, "cpu", reach_body_id=36, contact_body_ids=(7, 52))
    with pytest.raises(PulseError, match="strike_body_ids"):
        SmplxStrikeTaskB200(4, "cpu", strike_body_ids=(36, 52), contact_body_ids=feet)
    with pytest.raises(PulseError, match="strike_body_ids"):
        SmplxStrikeTaskB200(4, "cpu", strike_body_ids=(-1,), contact_body_ids=feet)
    for cls, kw in ((SmplxReachTaskB200, dict(reach_body_id=36)), (SmplxStrikeTaskB200, dict(strike_body_ids=(35, 36)))):
        for opt in ("power_reward", "power_usage_reward"):
            with pytest.raises(PulseError, match="power"):
                cls(4, "cpu", contact_body_ids=feet, **kw, **{opt: True})
    r = SmplxReachTaskB200(4, "cpu", reach_body_id=45, contact_body_ids=(7, 3, 40))
    s = SmplxStrikeTaskB200(4, "cpu", strike_body_ids=(35, 36, 45), contact_body_ids=feet)
    assert (r.layout, r.obs_size, r.reach_body_id, r.contact_body_mask) == ("smplx", 781, 45, (1 << 7) | (1 << 3) | (1 << 40))
    assert (s.layout, s.obs_size, s.strike_body_mask) == ("smplx", 793, (1 << 35) | (1 << 36) | (1 << 45))
    rb = torch.zeros(4, 52, 13)
    with pytest.raises(PulseError, match="dof_force"):
        r.post_physics_step(rb, torch.zeros(4, dtype=torch.int64), dof_force=torch.zeros(4, 153))
    with pytest.raises(PulseError, match="dof_force"):
        s.post_physics_step(rb, torch.zeros(4, dtype=torch.int64), torch.zeros(4, 13), torch.zeros(4, 3), dof_force=torch.zeros(4, 153))
    with pytest.raises(PulseError, match="52"):
        r.post_physics_step(torch.zeros(4, 24, 13), torch.zeros(4, dtype=torch.int64))
