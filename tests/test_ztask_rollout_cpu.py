"""CPU-side checks of the latent-task rollout's C boundary and of `ZTaskStepsB200`'s construction-time validation: struct layouts
against the header (gcc), exported symbols, rejected argument blocks, mismatched pieces, and the Philox index plane of the
`_update_task` draws.  No compute is attempted."""
import ctypes as C
import os
import re
import subprocess
import tempfile
from types import SimpleNamespace as NS

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("pulse_latent_post", "pulse_ztask_pre_physics", "pulse_reach_rollout_step", "pulse_ztask_rollout_step")


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def test_new_struct_sizes_match_header():
    from pulse_b200 import _lib
    src = ('#include <stdio.h>\n#include "pulse_b200.h"\nint main(){printf("%zu %zu\\n", sizeof(pulse_latent_post_args_t), '
           'sizeof(pulse_ztask_pre_physics_args_t));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [C.sizeof(_lib.LatentPostArgs), C.sizeof(_lib.ZTaskPrePhysicsArgs)]


def test_new_symbols_resolve(lib):
    from pulse_b200 import _lib
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    assert lib.pulse_abi_version() == 3


def test_entry_points_reject_bad_arguments(lib):
    from pulse_b200 import _lib
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    assert lib.pulse_latent_post(None, 4, None) == -1 and b"null" in lib.pulse_last_error()
    a = _lib.LatentPostArgs(mu=ptr, ld_mu=32, logstd=ptr, actions=ptr, ld_actions=32, neglogp=ptr, ld_neglogp=1, value=ptr, ld_value=1,
                            values_out=ptr, ld_values=1, prior_mu=ptr, ld_prior=64, z_bf16=ptr, ld_z=16, latent=32)
    assert lib.pulse_latent_post(C.byref(a), 4, None) == -1 and b"leading dimensions" in lib.pulse_last_error()
    a.ld_z, a.latent = 64, 200
    assert lib.pulse_latent_post(C.byref(a), 4, None) == -1 and b"latent" in lib.pulse_last_error()
    a.latent, a.prior_mu = 32, None
    assert lib.pulse_latent_post(C.byref(a), 4, None) == -1 and b"prior_mu" in lib.pulse_last_error()
    p = _lib.ZTaskPrePhysicsArgs(kind=9)
    assert lib.pulse_ztask_pre_physics(C.byref(p), 4, None) == -1 and b"unknown task kind" in lib.pulse_last_error()
    p = _lib.ZTaskPrePhysicsArgs(kind=_lib.ZTASK_SPEED, dofs=69, action=ptr, ld_action=69, pd_offset=ptr, pd_scale=ptr, pd_out=ptr, ld_pd=69)
    assert lib.pulse_ztask_pre_physics(C.byref(p), 4, None) == -1 and b"root_states" in lib.pulse_last_error()
    p.kind = _lib.ZTASK_REACH
    assert lib.pulse_ztask_pre_physics(C.byref(p), 4, None) == -1 and b"change_steps" in lib.pulse_last_error()
    p.progress_buf = p.change_steps = p.tar_pos = ptr
    assert lib.pulse_ztask_pre_physics(C.byref(p), 4, None) == -1 and b"randint" in lib.pulse_last_error()
    assert lib.pulse_reach_rollout_step(None, ptr, 4, None) == -1
    r = _lib.ReachStepArgs(body_state=ptr, body_env_stride=24 * 13, tar_pos=ptr, progress_buf=ptr, obs_buf=ptr, obs_stride=300, rew_buf=ptr,
                           reset_buf=ptr, terminate_buf=ptr, reach_body_id=23)
    assert lib.pulse_reach_rollout_step(C.byref(r), ptr, 4, None) == -1 and b"stride" in lib.pulse_last_error()
    assert lib.pulse_reach_rollout_step(C.byref(r), None, 4, None) == -1 and b"dones" in lib.pulse_last_error()
    za = _lib.ZTaskStepArgs(kind=7)
    assert lib.pulse_ztask_rollout_step(C.byref(za), ptr, 4, None) == -1 and b"unknown task kind" in lib.pulse_last_error()


def _pieces(kind="reach", reset_kind=None, task_w=None, policy_w=None, A=32, E=32, S=358, dof=69, disc=None):
    from pulse_b200 import _lib
    code = {"reach": _lib.ZTASK_REACH, "speed": _lib.ZTASK_SPEED, "strike": _lib.ZTASK_STRIKE}[kind]
    W = 373 if kind == "strike" else 361
    task = NS(kind=code, obs_size=W if task_w is None else task_w, num_envs=4)
    reset = NS(kind=kind if reset_kind is None else reset_kind)
    policy = NS(obs_size=W if policy_w is None else policy_w, A=A, disc=disc, device="cpu")
    vae = NS(E=E, S=S, A=dof)
    return task, reset, policy, vae


def test_constructor_rejects_mismatched_pieces():
    from pulse_b200 import PulseError, ZTaskStepsB200
    from pulse_b200.ztask_rollout import check_pieces
    for kind in ("reach", "speed", "strike"):
        assert check_pieces(*_pieces(kind)) == kind
    bad = [_pieces("reach", reset_kind="speed"),            # kinds differ
           _pieces("strike", policy_w=361),                  # the strike observation has 373 floats
           _pieces("speed", task_w=373),
           _pieces("reach", A=69),                           # the policy does not act in the VAE's latent
           _pieces("reach", E=64),
           _pieces("reach", S=934),
           _pieces("reach", disc=object())]
    for pieces in bad:
        with pytest.raises(PulseError):
            ZTaskStepsB200(*pieces, sim={})
    t, r, p, v = _pieces("reach")
    with pytest.raises(PulseError):
        ZTaskStepsB200(NS(obs_size=361), r, p, v, sim={})    # not a latent-task step object
    with pytest.raises(PulseError, match="sim lacks"):
        ZTaskStepsB200(t, r, p, v, sim={"body_state": None})


def test_update_task_plane_is_distinct_and_documented():
    """The `_update_task` draws sit on their own Philox index plane: it differs from the three the reset documents, the binding, the
    kernel and the header's draw table agree on it, and an env count below 2^31 cannot carry one plane into another."""
    from pulse_b200 import _lib
    planes = [_lib.ZTASK_PLANE_RESET, _lib.ZTASK_PLANE_STRIKE, _lib.ZTASK_PLANE_RESET_TASK, _lib.ZTASK_PLANE_UPDATE_TASK]
    assert planes[:3] == [0, 2 ** 32, 2 ** 33]
    assert len(set(planes)) == 4
    spans = sorted(planes)
    assert all(b - a >= 2 ** 31 for a, b in zip(spans, spans[1:]))
    cu = open(os.path.join(ROOT, "pulse_b200", "csrc", "ztask_rollout.cu")).read()
    m = re.search(r"kUpdateStream\s*=\s*(\d+)ull\s*<<\s*(\d+)", cu)
    assert m and int(m.group(1)) << int(m.group(2)) == _lib.ZTASK_PLANE_UPDATE_TASK
    rs = open(os.path.join(ROOT, "pulse_b200", "csrc", "ztask_reset.cu")).read()
    got = {int(a) << int(b) for a, b in re.findall(r"k(?:Strike|Task)Stream\s*=\s*(\d+)ull\s*<<\s*(\d+)", rs)}
    assert got == {_lib.ZTASK_PLANE_STRIKE, _lib.ZTASK_PLANE_RESET_TASK}
    hdr = open(os.path.join(ROOT, "include", "pulse_b200.h")).read()
    assert "index e + 3 * 2^32" in hdr and "index e + 2^33" in hdr and "index e + 2^32" in hdr
