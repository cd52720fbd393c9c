"""CPU-side checks of the C-ABI boundary: the library builds/loads and exports every symbol the
header declares; argument validation works without a GPU (no compute is attempted here)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "pulse_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(pulse_[a-z0-9_]+)\s*\(", txt)))


def test_header_symbols_exported(lib):
    from pulse_b200 import _lib
    names = _declared_symbols()
    assert len(names) >= 10
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/pulse_b200.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in pulse_b200/_lib.py"
    assert lib.pulse_abi_version() == 3


def test_struct_sizes_match_header(lib):
    """ctypes mirrors must have the C layout: compile a tiny C program with gcc and compare sizeof."""
    import subprocess
    import tempfile
    from pulse_b200 import _lib
    src = '#include <stdio.h>\n#include "pulse_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(pulse_motionlib_desc_t), sizeof(pulse_motion_query_t), sizeof(pulse_im_step_args_t), sizeof(pulse_amp_obs_args_t), sizeof(pulse_gae_args_t), sizeof(pulse_gemm_epilogue_t), sizeof(pulse_ppo_loss_args_t), sizeof(pulse_vae_latent_args_t), sizeof(pulse_reach_step_args_t), sizeof(pulse_loader_args_t), sizeof(pulse_reset_args_t), sizeof(pulse_policy_post_args_t), sizeof(pulse_amp_row_args_t), sizeof(pulse_peer_adam_args_t), sizeof(pulse_eval_args_t), sizeof(pulse_task_obs_args_t), sizeof(pulse_ztask_step_args_t));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [C.sizeof(_lib.MotionLibDesc), C.sizeof(_lib.MotionQuery), C.sizeof(_lib.ImStepArgs), C.sizeof(_lib.AmpObsArgs),
                     C.sizeof(_lib.GaeArgs), C.sizeof(_lib.GemmEpilogue), C.sizeof(_lib.PpoLossArgs), C.sizeof(_lib.VaeLatentArgs),
                     C.sizeof(_lib.ReachStepArgs), C.sizeof(_lib.LoaderArgs), C.sizeof(_lib.ResetArgs), C.sizeof(_lib.PolicyPostArgs),
                     C.sizeof(_lib.AmpRowArgs), C.sizeof(_lib.PeerAdamArgs), C.sizeof(_lib.EvalArgs), C.sizeof(_lib.TaskObsArgs), C.sizeof(_lib.ZTaskStepArgs)]


def test_argument_validation_without_gpu(lib):
    from pulse_b200 import _lib
    assert lib.pulse_im_step(None, None, 4, None) == -1
    assert b"null" in lib.pulse_last_error()
    assert lib.pulse_motion_state(None, None, 1, None) == -1
    assert lib.pulse_gae(None, 32, 8, None) == -1
    ta = _lib.TaskObsArgs(version=5, num_track=24, time_steps=1)
    assert lib.pulse_im_task_obs(C.byref(ta), None) == -1 and b"unsupported observation version" in lib.pulse_last_error()
    assert [lib.pulse_task_obs_size(v, 24, 1) for v in (1, 2, 3, 6, 7, 8, 9, 4)] == [360, 429, 216, 576, 216, 720, 438, -1]
    ta.version, ta.time_steps, ta.num_envs = 8, 3, 4
    assert lib.pulse_im_task_obs(C.byref(ta), None) == -1 and b"time_steps = 1" in lib.pulse_last_error()
    za = _lib.ZTaskStepArgs(kind=7)
    assert lib.pulse_ztask_step(C.byref(za), 4, None) == -1 and b"unknown task kind" in lib.pulse_last_error()
    ea = _lib.EvalArgs()
    assert lib.pulse_eval_step(C.byref(ea), None) == -1 and b"num_envs" in lib.pulse_last_error()
    pa = _lib.PeerAdamArgs()
    assert lib.pulse_peer_reduce_adam(None, None) == -1
    assert lib.pulse_peer_reduce_adam(C.byref(pa), None) == -1 and b"world" in lib.pulse_last_error()
    pa.world, pa.rank, pa.count = 2, 0, 6
    assert lib.pulse_peer_reduce_adam(C.byref(pa), None) == -1 and b"multiple of 4" in lib.pulse_last_error()
    a = _lib.GaeArgs()
    assert lib.pulse_gae(C.byref(a), 0, 8, None) == -1 and b"horizon" in lib.pulse_last_error()
    d = _lib.MotionLibDesc()
    h = C.c_void_p()
    assert lib.pulse_motionlib_create(C.byref(d), None, C.byref(h)) == -1
    with pytest.raises(_lib.PulseError):
        _lib.check(-1, "demo")


def test_no_cpu_fallback():
    """The product path refuses to run without a CUDA device instead of falling back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pulse_b200 import PulseError
    from pulse_b200.motion_lib import MotionLibB200
    from tests.helpers import load_npz
    with pytest.raises(PulseError):
        MotionLibB200.from_tables(load_npz("motionlib.npz"))


def test_product_does_not_import_oracle():
    import glob
    for f in glob.glob(os.path.join(ROOT, "pulse_b200", "**", "*.py"), recursive=True):
        src = open(f).read()
        assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S).replace("# oracle", ""), f"{f} references oracle/"


def test_new_entry_points_validate_arguments_without_gpu(lib):
    """Rows a14 / a19 / a20: the VAE / teacher / reach / PD entry points reject bad arguments before any launch."""
    from pulse_b200 import _lib
    assert lib.pulse_vae_latent_loss(None, 8, None) == -1 and b"null" in lib.pulse_last_error()
    a = _lib.VaeLatentArgs()
    assert lib.pulse_vae_latent_loss(C.byref(a), 8, None) == -1
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    a = _lib.VaeLatentArgs(enc_head=ptr, ld_enc=8, prior_head=ptr, ld_prior=8, noise=ptr, ld_noise=4, d_enc_head=ptr, ld_de=8,
                           d_prior_head=ptr, ld_dp=8, stats=ptr, latent=64, horizon=4)
    assert lib.pulse_vae_latent_loss(C.byref(a), 8, None) == -1 and b"latent" in lib.pulse_last_error()
    a.latent, a.progress, a.ar1_coef, a.horizon = 4, ptr, 0.005, 3
    assert lib.pulse_vae_latent_loss(C.byref(a), 8, None) == -1 and b"horizon" in lib.pulse_last_error()
    assert lib.pulse_vae_reparam(ptr, 8, None, 0, 4, 4, _lib.Z_SAMPLE, 1, -5.0, 2.0, ptr, 8, None, 0, None) == -1   # noise required
    assert lib.pulse_vae_reparam(ptr, 8, ptr, 4, 4, 4, 7, 1, -5.0, 2.0, ptr, 8, None, 0, None) == -1 and b"mode" in lib.pulse_last_error()
    assert lib.pulse_vae_action_loss(ptr, 200, ptr, 200, 4, 200, ptr, 200, 0, ptr, None) == -1               # > 128 actions
    assert lib.pulse_copy_cols_bf16(ptr, 7, 4, 6, ptr, 8, None, 0, None) == -1 and b"even" in lib.pulse_last_error()
    assert lib.pulse_normalize_cols(ptr, 8, 4, 8, ptr, None, 0.0, ptr, 8, 8, None) == -1                     # mean without rstd
    assert lib.pulse_pnn_compose(ptr, 64, 4, ptr, 2, _lib.ACT_SILU, 4, 8, 3, ptr, 8, None) == -1             # ld_a < num_actions
    assert lib.pulse_pd_targets(ptr, 4, ptr, ptr, None, 4, 8, ptr, 8, None) == -1                            # ld_a < dofs
    assert lib.pulse_reach_step(None, 4, None) == -1
    r = _lib.ReachStepArgs(body_state=ptr, body_env_stride=24 * 13, tar_pos=ptr, progress_buf=ptr, obs_buf=ptr, obs_stride=300, rew_buf=ptr,
                           reset_buf=ptr, terminate_buf=ptr, reach_body_id=23)
    assert lib.pulse_reach_step(C.byref(r), 4, None) == -1 and b"stride" in lib.pulse_last_error()
    r.obs_stride, r.reach_body_id = 361, 30
    assert lib.pulse_reach_step(C.byref(r), 4, None) == -1 and b"reach_body_id" in lib.pulse_last_error()
    r.reach_body_id, r.enable_early_termination = 23, 1
    assert lib.pulse_reach_step(C.byref(r), 4, None) == -1 and b"termination_heights" in lib.pulse_last_error()
    assert lib.pulse_reach_update_task(ptr, ptr, ptr, ptr, None, 1.0, 0.5, 1.5, 4, None) == -1


def test_reset_entry_point_validates_arguments_without_gpu(lib):
    """pulse_reset_ref_state (row a13 / 8f-3) rejects incomplete argument blocks before any launch."""
    from pulse_b200 import _lib
    assert lib.pulse_reset_ref_state(None, None, 4, None) == -1 and b"null" in lib.pulse_last_error()
    buf = (C.c_float * 256)()
    ptr = C.cast(buf, C.c_void_p)
    fake_lib = C.cast((C.c_char * 256)(), C.c_void_p)
    a = _lib.ResetArgs()
    assert lib.pulse_reset_ref_state(fake_lib, C.byref(a), 4, None) == -1 and b"mask" in lib.pulse_last_error()
    a.reset_buf = ptr
    assert lib.pulse_reset_ref_state(fake_lib, C.byref(a), 4, None) == -1 and b"env_list" in lib.pulse_last_error()
    a.env_list, a.count = ptr, ptr
    assert lib.pulse_reset_ref_state(fake_lib, C.byref(a), 4, None) == -1 and b"task buffer" in lib.pulse_last_error()
    a.motion_ids = a.motion_start_times = a.motion_start_offset = a.global_offset = a.progress_buf = ptr
    a.root_states = a.dof_pos = a.dof_vel = ptr
    a.root_env_stride, a.dof_env_stride, a.dof_elem_stride = 5, 138, 2
    assert lib.pulse_reset_ref_state(fake_lib, C.byref(a), 4, None) == -1 and b"strides" in lib.pulse_last_error()
    a.root_env_stride = 13
    a.amp_obs_buf, a.num_amp_steps = ptr, 40
    assert lib.pulse_reset_ref_state(fake_lib, C.byref(a), 4, None) == -1 and b"num_amp_steps" in lib.pulse_last_error()
