"""CPU checks of the distillation rollout's C entry points (`pulse_vae_reparam_philox`, `pulse_distill_pre_physics`): exported and bound,
the ABI version unchanged, and every bad argument refused with an error before anything is launched."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def test_symbols_exported_and_abi_unchanged(lib):
    from pulse_b200 import _lib
    for name in ("pulse_vae_reparam_philox", "pulse_distill_pre_physics"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    assert lib.pulse_abi_version() == 3 and _lib.ABI_VERSION == 3


def _host(n=4096):
    buf = (C.c_float * n)()
    return C.cast(buf, C.c_void_p), buf


def test_reparam_philox_rejects_bad_arguments(lib):
    from pulse_b200 import _lib
    p, _keep = _host()
    err = lambda: lib.pulse_last_error()

    def call(head=p, ld_head=64, rows=8, latent=32, ld_z=448, noise=None, ld_noise=0, z=p):
        return lib.pulse_vae_reparam_philox(head, ld_head, rows, latent, 1, -5.0, 2.0, 7, None, 0, z, ld_z, noise, ld_noise, None)

    assert call(head=None) == -1 and b"null" in err()
    assert call(z=None) == -1 and b"null" in err()
    assert call(rows=-1) == -1 and b"negative rows" in err()
    assert call(latent=33, ld_head=66) == -1 and b"latent 33" in err()
    assert call(latent=0) == -1 and b"latent 0" in err()
    assert call(ld_head=63) == -1 and b"stride too small" in err()
    assert call(ld_z=31) == -1 and b"stride too small" in err()
    assert call(noise=p, ld_noise=31) == -1 and b"noise_out row stride" in err()
    assert call(rows=0) == 0                     # nothing to do: returns before any launch
    with pytest.raises(_lib.PulseError, match="latent 40"):
        _lib.check(call(latent=40, ld_head=80), "pulse_vae_reparam_philox")


def test_pre_physics_rejects_bad_arguments(lib):
    from pulse_b200 import _lib
    p, _keep = _host()
    err = lambda: lib.pulse_last_error()

    def call(mus=p, ld_mus=69 * 32, off=p, scale=p, pd=p, ld_pd=69, prog=p, kin=p, ld_kin=32, rc=p, rows=8, dofs=69):
        return lib.pulse_distill_pre_physics(mus, ld_mus, off, scale, None, rows, dofs, pd, ld_pd, prog, kin, ld_kin, rc, None)

    for kw in (dict(mus=None), dict(off=None), dict(scale=None), dict(pd=None)):
        assert call(**kw) == -1 and b"null mus" in err(), kw
    for kw in (dict(prog=None), dict(kin=None), dict(rc=None)):
        assert call(**kw) == -1 and b"null progress_buf" in err(), kw
    assert call(rows=-3) == -1 and b"negative rows" in err()
    assert call(dofs=0) == -1 and b"dofs 0" in err()
    for kw in (dict(ld_mus=68), dict(ld_pd=68), dict(ld_kin=0)):
        assert call(**kw) == -1 and b"row strides too small" in err(), kw
    assert call(rows=0) == 0
    with pytest.raises(_lib.PulseError, match="negative rows"):
        _lib.check(call(rows=-1), "pulse_distill_pre_physics")


def test_driver_module_imports_without_gpu():
    """The host layer imports on a machine without a GPU (it raises only when used)."""
    from pulse_b200 import distill
    from pulse_b200.rollout import GraphRunner, PlayStepsB200
    assert issubclass(distill.DistillStepsB200, GraphRunner) and issubclass(PlayStepsB200, GraphRunner)
    assert set(distill.GETUP_KEYS) >= {"recovery_counter", "available_fall_states", "fall_id_assignments", "recovery_steps"}
