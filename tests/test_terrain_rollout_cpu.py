"""CPU-side checks of the terrain rollout's C boundary and of `TerrainStepsB200`'s construction-time validation: the new symbol, rejected
argument blocks of `pulse_terrain_rollout_step`, mismatched pieces, and the Philox blocks a horizon reads.  No compute is attempted."""
import ctypes as C
from types import SimpleNamespace as NS

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def test_new_symbol_resolves(lib):
    from pulse_b200 import TerrainStepsB200, _lib  # noqa: F401
    assert hasattr(lib, "pulse_terrain_rollout_step") and "pulse_terrain_rollout_step" in _lib.SIGNATURES
    assert lib.pulse_abi_version() == 3


def _args(ptr):
    from pulse_b200 import _lib
    return _lib.TerrainStepArgs(flags=_lib.STEP_ALL, body_state=ptr, body_env_stride=26 * 13, root_states=ptr, root_env_stride=26,
                                progress_buf=ptr, max_episode_length=300, contact_forces=ptr, contact_env_stride=26 * 3,
                                enable_early_termination=1, num_traj_samples=10, num_height_points=1024, num_center_points=9, head_body_id=13,
                                dt=1 / 30, traj_dur=10.1, traj_verts=ptr, height_points=ptr, center_points=ptr, obs_buf=ptr, obs_stride=1402,
                                rew_buf=ptr, reset_buf=ptr, terminate_buf=ptr)


def test_rollout_step_rejects_bad_arguments(lib):
    from pulse_b200 import _lib
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    dones = C.cast(buf, C.c_void_p)
    assert lib.pulse_terrain_rollout_step(None, dones, 4, None) == -1 and b"null" in lib.pulse_last_error()
    a = _args(ptr)
    assert lib.pulse_terrain_rollout_step(C.byref(a), None, 4, None) == -1 and b"dones" in lib.pulse_last_error()
    cases = [("flags", _lib.STEP_OBS, b"PULSE_STEP_ALL"), ("body_state", None, b"null input buffer"), ("progress_buf", None, b"null input buffer"),
             ("traj_verts", None, b"null input buffer"), ("rew_buf", None, b"rew_buf"), ("reset_buf", None, b"reset_buf"),
             ("obs_buf", None, b"obs_buf"), ("contact_forces", None, b"contact_forces"), ("body_env_stride", 23 * 13, b"strides too small"),
             ("root_env_stride", 12, b"strides too small"), ("obs_stride", 1401, b"obs_stride"), ("contact_env_stride", 71, b"contact_forces")]
    for field, value, msg in cases:
        a = _args(ptr)
        setattr(a, field, value)
        assert lib.pulse_terrain_rollout_step(C.byref(a), dones, 4, None) == -1, field
        err = lib.pulse_last_error()
        assert msg in err and b"pulse_terrain_rollout_step" in err, (field, err)
    a = _args(ptr)
    a.env_ids = ptr
    assert lib.pulse_terrain_rollout_step(C.byref(a), dones, 4, None) == -1
    assert lib.pulse_terrain_rollout_step(C.byref(_args(ptr)), dones, 0, None) == -1 and b"num_envs" in lib.pulse_last_error()


def _pieces(lib, plane=False, reset_hf=None, reset_scale=0.1, policy_cls=True, S=358, task_in=1044, A=32, E=32, vae_S=358, dof=69, disc=None):
    from pulse_b200.sept import SeptPolicy
    from pulse_b200.terrain import PedestrianTerrainTaskB200, TerrainB200
    from pulse_b200.terrain_reset import TerrainResetB200
    hf = torch.zeros(8, 8, dtype=torch.int16)
    terrain = TerrainB200(None if plane else hf, device="cpu")
    task = PedestrianTerrainTaskB200(4, device="cpu", terrain=terrain)
    reset = TerrainResetB200.__new__(TerrainResetB200)            # the fields the check reads; no MotionLib on the CPU
    reset.terrain = terrain if reset_hf is None else TerrainB200(reset_hf(hf.clone()), horizontal_scale=reset_scale, device="cpu")   # own upload
    policy = SeptPolicy.__new__(SeptPolicy) if policy_cls else NS()
    policy.S, policy.task_in, policy.A, policy.disc, policy.device = S, task_in, A, disc, "cpu"
    vae = NS(S=vae_S, E=E, A=dof)
    return task, reset, policy, vae


def _raised(hf):
    hf[3, 4] += 1
    return hf


def test_constructor_rejects_mismatched_pieces(lib):
    from pulse_b200 import PulseError, TerrainStepsB200
    from pulse_b200.terrain_rollout import check_pieces
    check_pieces(*_pieces(lib))
    check_pieces(*_pieces(lib, reset_hf=lambda hf: hf))           # a separate upload of the same map is the same heightfield
    bad = {"plane": dict(plane=True), "heightfield": dict(reset_hf=_raised),
           "different heightfields": dict(reset_hf=lambda hf: hf, reset_scale=0.2),
           "SeptPolicy": dict(policy_cls=False),
           "observation floats": dict(task_in=1040), "self observation": dict(S=356, task_in=1046), "VAE": dict(vae_S=934),
           "latent": dict(A=69), "latent has": dict(E=64), "69 dof": dict(dof=72), "discriminator": dict(disc=object())}
    for msg, kw in bad.items():
        with pytest.raises(PulseError, match=msg):
            TerrainStepsB200(*_pieces(lib, **kw), sim={})
    t, r, p, v = _pieces(lib)
    with pytest.raises(PulseError, match="PedestrianTerrainTaskB200"):
        TerrainStepsB200(NS(terrain=t.terrain, get_obs_size=lambda: 1402), r, p, v, sim={})
    with pytest.raises(PulseError, match="TerrainResetB200"):
        TerrainStepsB200(t, NS(terrain=t.terrain), p, v, sim={})
    sim = {k: torch.zeros(4) for k in ("body_state", "root_states", "dof_pos", "dof_vel", "progress_buf", "sampled_motion_ids", "motion_start_times")}
    with pytest.raises(PulseError, match="contact_forces"):          # early termination is on by default
        TerrainStepsB200(t, r, p, v, sim=sim)
    t.power_reward = True
    with pytest.raises(PulseError, match="dof_force"):
        TerrainStepsB200(t, r, p, v, sim=dict(sim, contact_forces=torch.zeros(4)))
    t.power_reward, t.enable_early_termination = False, False
    with pytest.raises(PulseError, match="sim has 5 envs"):
        TerrainStepsB200(t, r, p, v, sim=dict(sim, progress_buf=torch.zeros(5)))


def test_philox_blocks_never_repeat_across_steps_and_horizons(lib):
    """Reset, location, trajectory and latent draws: over three horizons of 32 steps (the policy's offset moving on by 32 after each),
    no Philox block is read twice, and the keying is the one the header documents (test_gpu_terrain_rollout.py regenerates these
    blocks on the host and checks them against the kernels' draws)."""
    from pulse_b200 import _lib
    from pulse_b200.terrain_rollout import philox_blocks
    T, n = 32, 1536
    seen = set()
    total = 0
    for env in (0, 1, 777, n - 1):
        for h in range(3):
            for t in range(T):
                blocks = philox_blocks(env, t, h * T)
                total += len(blocks)
                seen.update(blocks)
    assert len(seen) == total
    b = philox_blocks(5, 3, 64)
    assert b[0] == ("reset", 5, 67)                                                  # pulse_reset_terrain: index e, counter offset
    assert b[1] == ("reset", 5 + 4 * 2 ** 32, _lib.TRAJ_VERTS * 67) and b[_lib.TRAJ_VERTS] == ("reset", 5 + 4 * 2 ** 32, _lib.TRAJ_VERTS * 68 - 1)
    assert b[_lib.TRAJ_VERTS + 1:] == [("policy", 5 * 64 + p, 67) for p in range(16)]
    hdr = open(_lib.__file__.replace("pulse_b200/_lib.py", "include/pulse_b200.h")).read()
    assert "index e + 4 * 2^32 pulse_traj_reset_list" in hdr and "pulse_terrain_rollout_step" in hdr


def test_host_philox_matches_the_known_answers():
    """tests/philox_ref.py, which the GPU tests use to regenerate the kernels' draws, against the Random123 known-answer vectors of
    Philox4x32-10 (counter words = index lo / hi, offset lo / hi; key = seed lo / hi)."""
    from tests.philox_ref import philox4x32_10
    kat = [((0, 0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((2 ** 64 - 1, 2 ** 64 - 1, 2 ** 64 - 1), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x299F31D0A4093822, 0x85A308D3243F6A88, 0x0370734413198A2E), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for (seed, index, offset), words in kat:
        assert tuple(int(w) for w in philox4x32_10(seed, index, offset)) == words
