"""CPU-side checks of the downstream tasks' PPO baseline (the dof-space policy of HumanoidReach / HumanoidSpeed / HumanoidStrike under
learning=ppo): the action-count bounds of `pulse_policy_post` and `pulse_ppo_loss` (checked before any launch), `check_pieces` with
`vae=None`, and the Philox index layout of `policy_post` at the SMPL-X policy's 153 actions.  No compute is attempted."""
import ctypes as C
import os
import re
from types import SimpleNamespace as NS

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def policy_post_index(rows: int, num_actions: int) -> np.ndarray:
    """The Philox block index of action pair p of row r, as pulse_b200.h documents it: r * 64 + p up to 128 actions, r * 128 + p above.
    Returns uint64 [rows, pairs]."""
    stride = 64 if num_actions <= 128 else 128
    pairs = (num_actions + 1) // 2
    return np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(stride) + np.arange(pairs, dtype=np.uint64)[None, :]


def policy_post_stride(num_actions: int) -> int:
    return 64 if num_actions <= 128 else 128


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def test_entry_points_take_up_to_256_actions(lib):
    """153 and 256 pass the action-count check (the next check, on the leading dimensions, is what refuses these argument blocks, so
    nothing is launched); 257 and 0 are refused.  rows > 0 throughout: a zero-row call returns before any check."""
    from pulse_b200 import _lib
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    err = lambda: lib.pulse_last_error().decode()
    for A in (69, 128, 129, 153, 256):
        a = _lib.PolicyPostArgs(mu=ptr, ld_mu=A - 1, logstd=ptr, actions=ptr, ld_actions=A, neglogp=ptr, ld_neglogp=1, num_actions=A)
        assert lib.pulse_policy_post(C.byref(a), 4, None) == -1 and "leading dimensions" in err(), (A, err())
        p = _lib.PpoLossArgs(mu=ptr, ld_mu=A - 1, value=ptr, ld_value=1, actions=ptr, old_neglogp=ptr, advantages=ptr, returns=ptr, logstd=ptr,
                             num_actions=A)
        assert lib.pulse_ppo_loss(C.byref(p), 4, None) == -1 and "leading dimensions" in err(), (A, err())
    for A in (0, 257, 512):
        a = _lib.PolicyPostArgs(mu=ptr, ld_mu=512, logstd=ptr, actions=ptr, ld_actions=512, neglogp=ptr, ld_neglogp=1, num_actions=A)
        assert lib.pulse_policy_post(C.byref(a), 4, None) == -1 and "outside [1,256]" in err(), (A, err())
        p = _lib.PpoLossArgs(mu=ptr, ld_mu=512, value=ptr, ld_value=1, actions=ptr, old_neglogp=ptr, advantages=ptr, returns=ptr, logstd=ptr,
                             num_actions=A)
        assert lib.pulse_ppo_loss(C.byref(p), 4, None) == -1 and "outside [1,256]" in err(), (A, err())
    a = _lib.PolicyPostArgs(mu=ptr, ld_mu=512, logstd=ptr, actions=ptr, ld_actions=512, neglogp=ptr, ld_neglogp=1, num_actions=257)
    assert lib.pulse_policy_post(C.byref(a), 0, None) == 0                      # no rows: nothing to check or launch


@pytest.mark.parametrize("A", [1, 69, 127, 128, 129, 153, 255, 256])
def test_policy_post_philox_blocks_are_disjoint(A):
    idx = policy_post_index(1000, A)
    assert np.unique(idx).size == idx.size, "two (row, pair) draws share a Philox block"
    if A <= 128:
        r, p = np.meshgrid(np.arange(1000, dtype=np.uint64), np.arange((A + 1) // 2, dtype=np.uint64), indexing="ij")
        assert np.array_equal(idx, r * np.uint64(64) + p)
    # the last block of row r lies below the first of row r + 1
    assert bool((idx[:-1, -1] < idx[1:, 0]).all())


def test_policy_post_layout_is_documented_and_implemented():
    """The header's table, the kernel's stride choice and the test's restatement agree."""
    hdr = open(os.path.join(ROOT, "include", "pulse_b200.h")).read()
    assert "num_actions <= 128        index r * 64 + p" in hdr and "128 < num_actions <= 256  index r * 128 + p" in hdr
    cu = open(os.path.join(ROOT, "pulse_b200", "csrc", "rollout_ops.cu")).read()
    m = re.search(r"row_blocks\s*=\s*A\s*<=\s*(\d+)\s*\?\s*(\d+)ull\s*:\s*(\d+)ull", cu)
    assert m and tuple(int(x) for x in m.groups()) == (128, 64, 128)
    assert "static_cast<unsigned long long>(row) * row_blocks" in cu
    assert [policy_post_stride(A) for A in (69, 128, 129, 153, 256)] == [64, 64, 128, 128, 128]


def _pieces(layout, kind, A, with_vae=False, E=None):
    from pulse_b200 import _lib
    code = {"reach": _lib.ZTASK_REACH, "speed": _lib.ZTASK_SPEED, "strike": _lib.ZTASK_STRIKE}[kind]
    W = {("smpl", "reach"): 361, ("smpl", "speed"): 361, ("smpl", "strike"): 373,
         ("smplx", "reach"): 781, ("smplx", "speed"): 781, ("smplx", "strike"): 793}[(layout, kind)]
    smplx = layout == "smplx"
    task = NS(kind=code, obs_size=W, num_envs=4, layout=layout)
    reset = NS(kind=kind, smplx=smplx, bodies=52 if smplx else 24)
    policy = NS(obs_size=W, A=A, disc=None, device="cpu")
    vae = None
    if with_vae:
        vae = NS(E=E if E is not None else (48 if smplx else 32), S=778 if smplx else 358, A=153 if smplx else 69)
    return task, reset, policy, vae


@pytest.mark.parametrize("kind", ["reach", "speed", "strike"])
@pytest.mark.parametrize("layout,dofs", [("smpl", 69), ("smplx", 153)])
def test_check_pieces_takes_the_dof_space_policy_without_a_vae(layout, dofs, kind):
    from pulse_b200 import PulseError, ZTaskStepsB200
    from pulse_b200.ztask_rollout import check_pieces
    assert check_pieces(*_pieces(layout, kind, dofs)) == kind
    # the latent driver is unchanged
    assert check_pieces(*_pieces(layout, kind, 48 if layout == "smplx" else 32, with_vae=True)) == kind
    latent = 48 if layout == "smplx" else 32
    with pytest.raises(PulseError, match=f"without a VAE the policy acts in the {layout} humanoid's {dofs} dofs, not in {latent}"):
        check_pieces(*_pieces(layout, kind, latent))                              # a latent-width policy without its VAE
    with pytest.raises(PulseError, match=f"acts in the {layout} humanoid's {dofs} dofs, but a VAE was given"):
        check_pieces(*_pieces(layout, kind, dofs, with_vae=True))                 # a dof-width policy with a VAE
    other = 153 if layout == "smpl" else 69
    with pytest.raises(PulseError, match=f"{dofs} dofs, not in {other}"):
        check_pieces(*_pieces(layout, kind, other))                               # the other layout's dofs
    with pytest.raises(PulseError):
        ZTaskStepsB200(*_pieces(layout, kind, latent), sim={})
    with pytest.raises(PulseError, match="sim lacks"):
        ZTaskStepsB200(*_pieces(layout, kind, dofs), sim={"body_state": None})
