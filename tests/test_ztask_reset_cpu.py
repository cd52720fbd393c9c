"""CPU checks of the latent-space tasks' reset: the oracle (tests/ztask_reset_oracle.py) against the unmodified reference's
`_reset_ref_state_init` / `_reset_target` / `_init_amp_obs` / `_reset_task` recorded in tests/golden/ztask_reset.npz, the per-frame
ground table against the reference's own ground-fix arithmetic, and the C ABI and argument checks of `pulse_reset_ztask` /
`pulse_ztask_reset_task`."""
import ctypes as C
import os
import types

import pytest
import torch

from tests import ztask_reset_oracle as zo
from tests.helpers import load_npz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"reach": ("reach", True, zo.RANDOM), "reach_start": ("reach", True, zo.START), "speed": ("speed", True, zo.RANDOM),
         "speed_tilted": ("speed", False, zo.RANDOM), "speed_start": ("speed", True, zo.START), "strike": ("strike", True, zo.RANDOM),
         "strike_start": ("strike", True, zo.START)}
N = 40


@pytest.fixture(scope="module")
def fx():
    return load_npz("ztask_reset.npz")


@pytest.fixture(scope="module")
def tables():
    from pulse_b200.ztask_reset import smpl_ground_table
    tb, betas = zo.fixture_tables()
    return tb, betas, smpl_ground_table(tb.motion_aa, zo.StandInParser(), betas)


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def injected(fx, case, kind, init):
    """The recorded draws in the per-env form the kernels take."""
    ids = fx[case + "_env_ids"]
    names = str(fx[case + "_draws"]).split()
    draws = [fx[f"{case}_draw{i}"] for i in range(len(names))]
    d = {"motion_ids": torch.zeros(N, dtype=torch.int64), "phase": torch.zeros(N), "strike_u": torch.zeros(N, 4)}
    d["motion_ids"][ids] = draws.pop(0)
    if init == zo.RANDOM:
        d["phase"][ids] = draws.pop(0)
    if kind == "strike":
        for c in range(4):
            d["strike_u"][ids, c] = draws.pop(0)
    else:
        d["task_u"], d["task_steps"] = draws.pop(0), draws.pop(0)
    assert not draws
    return ids, d


def zero_state(kind):
    st = {"root_states": torch.zeros(N, 13), "dof_pos": torch.zeros(N, 69), "dof_vel": torch.zeros(N, 69), "body_state": torch.zeros(N, 24, 13),
          "sampled_motion_ids": torch.zeros(N, dtype=torch.int64), "motion_start_times": torch.zeros(N),
          "progress_buf": torch.zeros(N, dtype=torch.int64), "reset_buf": torch.zeros(N, dtype=torch.int64),
          "terminate_buf": torch.zeros(N, dtype=torch.int64), "contact_forces": torch.zeros(N, 24, 3), "amp_obs_buf": torch.zeros(N, 10, 195)}
    if kind == "strike":
        st["target_states"] = torch.zeros(N, 13)
    return st


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reproduces_reference_reset(fx, tables, case):
    """Clips and start times exactly, states, AMP rows and the strike target within 2e-6 of the reference, which lifts each pose with
    the parser's mesh instead of the floor table; the reach / speed task draws exactly."""
    kind, upright, init = CASES[case]
    tb, _, floor = tables
    ids, d = injected(fx, case, kind, init)
    o = zo.ztask_reset(tb, zero_state(kind), ids, d, floor, kind, upright=upright, state_init=init, num_amp_steps=10, width=195)
    assert torch.equal(o["sampled_motion_ids"], fx[case + "_motion_ids"])
    assert torch.equal(o["motion_start_times"], fx[case + "_start_times"])
    for k, ref in (("root_states", "root_states"), ("dof_pos", "dof_pos"), ("dof_vel", "dof_vel"), ("body_state", "body_state"),
                   ("amp_obs_buf", "amp_obs")) + ((("target_states", "target_states"),) if kind == "strike" else ()):
        torch.testing.assert_close(o[k], fx[case + "_" + ref], rtol=0, atol=2e-6, msg=lambda m: f"{case} {k}: {m}")
    if kind == "reach":
        tar, change = zo.reach_task(d["task_u"], d["task_steps"], fx[case + "_progress"][ids], **zo.REACH)
        assert torch.equal(tar, fx[case + "_tar_pos"][ids]) and torch.equal(change, fx[case + "_change_steps"][ids])
    elif kind == "speed":
        spd, change = zo.speed_task(d["task_u"], d["task_steps"], fx[case + "_progress"][ids], **zo.SPEED)
        assert torch.equal(spd, fx[case + "_tar_speed"][ids]) and torch.equal(change, fx[case + "_change_steps"][ids])


def test_fixture_covers_the_edge_cases(fx):
    """Zero-weight clips are never drawn, the tilted speed case really has a non-upright heading, and the strike draws hit both the
    near and the far branch."""
    prob = fx["prob"]
    for case in CASES:
        assert bool((prob[fx[case + "_motion_ids"][fx[case + "_env_ids"]]] > 0).all())
    near = fx["strike_draw2"]
    assert bool((near < zo.STRIKE["near_prob"]).any()) and bool((near >= zo.STRIKE["near_prob"]).any())
    assert not torch.allclose(fx["speed_tilted_root_states"], fx["speed_root_states"])


def test_ground_table_matches_the_reference_lift(tables):
    """`floor(f) + root_z - 0.02` equals the reference's `min_v (V - (J0 - root)).z - 0.02` with the mesh at the root's translation,
    to a few ulp (the order of the additions differs)."""
    tb, betas, floor = tables
    parser = zo.StandInParser()
    root = torch.randn(tb.motion_aa.shape[0], 3, generator=torch.Generator().manual_seed(3)) + torch.tensor([0.0, 0.0, 0.9])
    V, J = parser.get_joints_verts(tb.motion_aa, betas.expand(root.shape[0], 10), root)
    ref = (V - (J[:, 0] - root)[:, None])[..., -1].min(dim=-1).values - 0.02
    torch.testing.assert_close(floor + root[:, 2] - 0.02, ref, rtol=0, atol=1e-6)
    assert float(floor.std()) > 1e-3                  # the lift depends on the pose


def test_ztask_reset_symbols_and_struct_layout(lib):
    import subprocess
    import tempfile
    from pulse_b200 import _lib
    for n in ("pulse_reset_ztask", "pulse_ztask_reset_task", "pulse_reach_obs_list", "pulse_ztask_obs_list"):
        assert hasattr(lib, n) and n in _lib.SIGNATURES
    assert lib.pulse_abi_version() == 3
    rf = ("motion_u", "sampling_cdf", "floor_len", "amp_width", "dt", "amp_obs_buf", "rigid_body_state", "contact_bodies", "target_states", "near_prob",
          "tar_dist_max", "tar_actor_ids", "tar_actor_list", "count")
    tf = ("count", "steps_in", "offset_dev", "tar_speed", "speed_min", "steps_min", "steps_max")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "pulse_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu", '
           'sizeof(pulse_ztask_reset_args_t), sizeof(pulse_ztask_task_args_t), sizeof(pulse_reset_args_t), sizeof(pulse_getup_reset_args_t), '
           'sizeof(pulse_ztask_step_args_t), sizeof(pulse_reach_step_args_t));'
           + "".join(f'printf(" %zu", offsetof(pulse_ztask_reset_args_t, {f}));' for f in rf)
           + "".join(f'printf(" %zu", offsetof(pulse_ztask_task_args_t, {f}));' for f in tf)
           + 'printf(" %d %d %d %d %d %d %d", PULSE_ZTASK_REACH, PULSE_ZPOSE_AS_IS, PULSE_ZPOSE_ROOT_XY_ZERO, PULSE_ZPOSE_FACE_X, '
             'PULSE_ZINIT_RANDOM, PULSE_ZINIT_START, PULSE_AMP_OBS_NO_HEIGHT); return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert got == ([C.sizeof(_lib.ZTaskResetArgs), C.sizeof(_lib.ZTaskTaskArgs), C.sizeof(_lib.ResetArgs), C.sizeof(_lib.GetupResetArgs),
                    C.sizeof(_lib.ZTaskStepArgs), C.sizeof(_lib.ReachStepArgs)]
                   + [getattr(_lib.ZTaskResetArgs, f).offset for f in rf] + [getattr(_lib.ZTaskTaskArgs, f).offset for f in tf]
                   + [_lib.ZTASK_REACH, _lib.ZPOSE_AS_IS, _lib.ZPOSE_ROOT_XY_ZERO, _lib.ZPOSE_FACE_X, _lib.ZINIT_RANDOM, _lib.ZINIT_START, 195])
    # the existing argument structs keep their sizes
    assert [C.sizeof(_lib.ResetArgs), C.sizeof(_lib.GetupResetArgs), C.sizeof(_lib.ZTaskStepArgs), C.sizeof(_lib.ReachStepArgs)] == got[2:6]


def _valid_reset_args(_lib, ptr):
    a = _lib.ZTaskResetArgs()
    a.reset_buf = a.env_list = a.count = ptr
    a.sampled_motion_ids = a.motion_start_times = a.progress_buf = ptr
    a.root_states = a.dof_pos = a.dof_vel = a.rigid_body_state = ptr
    a.root_env_stride, a.dof_env_stride, a.dof_elem_stride, a.body_env_stride = 13, 138, 2, 312
    a.floor, a.floor_len, a.sampling_cdf = ptr, 10, ptr
    return a


def test_ztask_entry_points_validate_arguments_without_gpu(lib):
    """Every refusal happens before anything touches the device, so a CPU-only machine exercises them all."""
    from pulse_b200 import _lib
    buf = (C.c_float * 256)()
    ptr = C.cast(buf, C.c_void_p)
    desc = _lib.MotionLibDesc(aux_rec=ptr, total_frames=10, num_motions=2)   # a handle is its descriptor (pulse_common.cuh)
    fake_lib = C.cast(C.pointer(desc), C.c_void_p)
    assert lib.pulse_reset_ztask(None, None, 4, None) == -1 and b"null" in lib.pulse_last_error()
    assert lib.pulse_reset_ztask(fake_lib, C.byref(_lib.ZTaskResetArgs()), 4, None) == -1 and b"mask" in lib.pulse_last_error()

    def refuses(change, words):
        a = _valid_reset_args(_lib, ptr)
        change(a)
        assert lib.pulse_reset_ztask(fake_lib, C.byref(a), 4, None) == -1
        assert words.encode() in lib.pulse_last_error(), lib.pulse_last_error()

    refuses(lambda a: setattr(a, "count", None), "count outputs")
    refuses(lambda a: setattr(a, "motion_start_times", None), "null task buffer")
    refuses(lambda a: setattr(a, "rigid_body_state", None), "null simulator tensor")
    refuses(lambda a: setattr(a, "body_env_stride", 300), "strides")
    refuses(lambda a: setattr(a, "dof_env_stride", 100), "strides")
    refuses(lambda a: (setattr(a, "contact_forces", ptr), setattr(a, "contact_bodies", 24), setattr(a, "contact_env_stride", 40)), "contact-force")
    refuses(lambda a: (setattr(a, "target_states", ptr), setattr(a, "target_env_stride", 7)), "target_states stride")
    refuses(lambda a: setattr(a, "floor_len", 9), "floor table of 9 frames")
    refuses(lambda a: setattr(a, "floor", None), "floor table")
    refuses(lambda a: setattr(a, "sampling_cdf", None), "sampling_cdf")
    refuses(lambda a: setattr(a, "pose_mode", 3), "pose_mode")
    refuses(lambda a: setattr(a, "state_init", 2), "state_init")
    refuses(lambda a: (setattr(a, "amp_obs_buf", ptr), setattr(a, "num_amp_steps", 10), setattr(a, "amp_width", 194)), "amp_width 194")
    refuses(lambda a: (setattr(a, "amp_obs_buf", ptr), setattr(a, "num_amp_steps", 17), setattr(a, "amp_width", 195)), "num_amp_steps")
    refuses(lambda a: (setattr(a, "env_ids_in", ptr), setattr(a, "num_ids", 5)), "num_ids")
    a = _valid_reset_args(_lib, ptr)
    assert lib.pulse_reset_ztask(fake_lib, C.byref(a), 0, None) == 0          # nothing to do: no launch
    a.sampling_cdf, a.motion_ids_in = None, ptr                                  # injected clips need no CDF
    assert lib.pulse_reset_ztask(fake_lib, C.byref(a), 0, None) == 0

    t = _lib.ZTaskTaskArgs(kind=_lib.ZTASK_STRIKE)
    assert lib.pulse_ztask_reset_task(C.byref(t), 4, None) == -1 and b"kind" in lib.pulse_last_error()
    t.kind = _lib.ZTASK_REACH
    assert lib.pulse_ztask_reset_task(C.byref(t), 4, None) == -1 and b"null list" in lib.pulse_last_error()
    t.env_list = t.count = t.progress_buf = t.change_steps = ptr
    assert lib.pulse_ztask_reset_task(C.byref(t), 4, None) == -1 and b"tar_pos" in lib.pulse_last_error()
    t.tar_pos = ptr
    assert lib.pulse_ztask_reset_task(C.byref(t), 4, None) == -1 and b"randint range" in lib.pulse_last_error()
    t.kind = _lib.ZTASK_SPEED
    assert lib.pulse_ztask_reset_task(C.byref(t), 4, None) == -1 and b"tar_speed" in lib.pulse_last_error()


def test_obs_list_entry_points_validate_arguments_without_gpu(lib):
    from pulse_b200 import _lib
    buf = (C.c_float * 256)()
    ptr = C.cast(buf, C.c_void_p)
    r = _lib.ReachStepArgs()
    assert lib.pulse_reach_obs_list(C.byref(r), None, ptr, 4, None) == -1 and b"env_list" in lib.pulse_last_error()
    assert lib.pulse_reach_obs_list(C.byref(r), ptr, ptr, 4, None) == -1 and b"null buffer" in lib.pulse_last_error()
    r.body_state = r.tar_pos = r.obs_buf = ptr
    r.body_env_stride, r.obs_stride = 312, 300
    assert lib.pulse_reach_obs_list(C.byref(r), ptr, ptr, 4, None) == -1 and b"strides" in lib.pulse_last_error()
    z = _lib.ZTaskStepArgs(kind=_lib.ZTASK_SPEED, body_state=ptr, obs_buf=ptr, body_env_stride=312, obs_stride=361)
    assert lib.pulse_ztask_obs_list(C.byref(z), ptr, ptr, 4, None) == -1 and b"tar_speed" in lib.pulse_last_error()
    z.kind, z.obs_stride = _lib.ZTASK_STRIKE, 373
    assert lib.pulse_ztask_obs_list(C.byref(z), ptr, ptr, 4, None) == -1 and b"target_states" in lib.pulse_last_error()
    z.kind = 9
    assert lib.pulse_ztask_obs_list(C.byref(z), ptr, ptr, 4, None) == -1 and b"kind" in lib.pulse_last_error()


@pytest.mark.parametrize("change,words", [
    (lambda t: setattr(t, "humanoid_type", "smplx"), "humanoid_type"),
    (lambda t: setattr(t, "amp_obs_v", 2), "amp_obs_v"),
    (lambda t: setattr(t, "_key_body_ids", torch.tensor([7, 3, 22, 18])), "keyBodies"),
    (lambda t: setattr(t, "_has_dof_subset", False), "dof_subset"),
    (lambda t: t.humanoid_shapes.__setitem__((3, 2), 0.5), "shape variation"),
])
def test_mixin_refuses_what_the_device_reset_does_not_serve(change, words):
    """Each refusal names the option; the checks run before anything touches the device."""
    from pulse_b200 import _lib
    from pulse_b200.ztask_reset import HumanoidZTaskResetB200Mixin
    from tests.ztask_standin import StandInZTask

    class Task(HumanoidZTaskResetB200Mixin, StandInZTask):
        pass

    t = Task("reach", types.SimpleNamespace(gts=None), "cpu", 8)
    change(t)
    with pytest.raises(_lib.PulseError, match=words):
        t._pulse_ztask_setup()


def test_mixin_serves_only_the_three_tasks():
    from pulse_b200 import _lib
    from pulse_b200.ztask_reset import HumanoidZTaskResetB200Mixin
    with pytest.raises(_lib.PulseError, match="HumanoidReach"):
        HumanoidZTaskResetB200Mixin()._pulse_ztask_kind()
