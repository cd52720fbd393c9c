"""CPU-side checks of the tracked-body imitation step and of `ImZStepsB200`'s construction: the new struct and symbol, every rejected
argument of `pulse_im_track_step`, every constructor refusal, the column map of the tracked row against the oracle's v6 / v7 of the
subset, and the Philox blocks a horizon reads.  No compute is attempted."""
import ctypes as C
from types import SimpleNamespace as NS

import pytest
import torch

TRACK_VR = (13, 18, 23)          # env_pulse_im.yaml trackBodies: Head, L_Hand, R_Hand


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def test_struct_and_symbol(lib):
    from pulse_b200 import ImZStepsB200, _lib  # noqa: F401
    assert C.sizeof(_lib.ImTrack) == 32
    assert [f for f, _ in _lib.ImTrack._fields_] == ["rank", "num_track", "version"]
    assert hasattr(lib, "pulse_im_track_step") and "pulse_im_track_step" in _lib.SIGNATURES
    assert lib.pulse_abi_version() == 3
    hdr = open(_lib.__file__.replace("pulse_b200/_lib.py", "include/pulse_b200.h")).read()
    assert "pulse_im_track_t" in hdr and "int pulse_im_track_step(" in hdr


def _track(ids, version=6):
    from pulse_b200 import _lib
    tr = _lib.ImTrack(num_track=len(ids), version=version)
    for j in range(24):
        tr.rank[j] = ids.index(j) if j in ids else -1
    return tr


def test_track_step_rejects_bad_arguments(lib):
    from pulse_b200 import _lib
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    desc = _lib.MotionLibDesc()                       # a zeroed MotionLib stands in for the handle: no check reaches its tables
    ml = C.c_void_p(C.addressof(desc))

    def args(obs_stride=430):
        return _lib.ImStepArgs(flags=_lib.STEP_OBS, body_state=ptr, body_env_stride=312, progress_buf=ptr, motion_ids=ptr,
                               motion_start_times=ptr, motion_start_offset=ptr, global_offset=ptr, obs_buf=ptr, obs_stride=obs_stride)

    def call(a, tr, n=4):
        return lib.pulse_im_track_step(ml, C.byref(a), None if tr is None else C.byref(tr), n, None)

    assert lib.pulse_im_track_step(None, C.byref(args()), C.byref(_track(list(TRACK_VR))), 4, None) == -1
    assert b"null lib/args" in lib.pulse_last_error()
    cases = [(None, b"null track")]
    for k in (0, 25):
        bad = _track(list(TRACK_VR))
        bad.num_track = k
        cases.append((bad, b"num_track %d outside [1, 24]" % k))
    dup = _track(list(TRACK_VR))
    dup.rank[5] = 1                                   # two bodies at rank 1
    high = _track(list(TRACK_VR))
    high.rank[23] = 3                                 # rank K with K = 3
    short = _track(list(TRACK_VR))
    short.rank[18] = -1                               # ranks 0 and 2 only
    cases += [(dup, b"not a permutation"), (high, b"not a permutation"), (short, b"not a permutation"),
              (_track(list(TRACK_VR), version=8), b"version 8")]
    for tr, msg in cases:
        assert call(args(), tr) == -1, msg
        err = lib.pulse_last_error()
        assert msg in err and err.startswith(b"pulse_im_track_step"), (msg, err)
    for ids, version, width in ((TRACK_VR, 6, 430), (TRACK_VR, 7, 385), ((4,), 7, 367), (tuple(range(24)), 6, 934)):
        assert call(args(width - 1), _track(list(ids), version)) == -1
        assert b"obs_stride < %d" % width in lib.pulse_last_error()
    a = args()
    a.body_env_stride = 311                           # the checks shared with pulse_im_step, named for this entry point
    assert call(a, _track(list(TRACK_VR))) == -1 and lib.pulse_last_error().startswith(b"pulse_im_track_step: body_env_stride")
    assert call(args(), _track(list(TRACK_VR)), n=-1) == -1 and b"negative num_envs" in lib.pulse_last_error()
    assert call(args(), _track(list(TRACK_VR)), n=0) == 0


def test_compute_tracked_configuration(lib):
    from pulse_b200 import PulseError
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    ml = NS(_device="cpu")
    assert HumanoidImCompute(ml).obs_size == 934 and HumanoidImCompute(ml).track is None
    comp = HumanoidImCompute(ml, ImConfig(track_body_ids=(23, 13, 18), obs_version=7))
    assert comp.obs_size == 358 + 27 and comp.track.num_track == 3 and comp.track.version == 7
    assert [comp.track.rank[j] for j in (13, 18, 23, 0)] == [1, 2, 0, -1]
    assert HumanoidImCompute(ml, ImConfig(track_body_ids=TRACK_VR)).obs_size == 430
    for ids, v, msg in (((13, 13), 6, "distinct"), ((24,), 6, "distinct"), ((), 6, "distinct"), (TRACK_VR, 8, "version 8")):
        with pytest.raises(PulseError, match=msg):
            HumanoidImCompute(ml, ImConfig(track_body_ids=ids, obs_version=v))


def _pieces(track=TRACK_VR, version=6, obs_size=430, A=32, E=32, vae_S=358, dof=69, disc=None, **cfg):
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    comp = HumanoidImCompute(NS(_device="cpu"), ImConfig(track_body_ids=track, obs_version=version, **cfg))
    policy = NS(obs_size=obs_size, A=A, disc=disc, device="cpu")
    return comp, policy, NS(S=vae_S, E=E, A=dof)


def test_constructor_refusals(lib):
    from pulse_b200 import ImZStepsB200, PulseError
    from pulse_b200.imz_rollout import SIM_KEYS, check_pieces
    check_pieces(*_pieces())
    check_pieces(*_pieces(version=7, obs_size=385))
    bad = {"tracked configuration": dict(track=None, obs_size=934), "cycle_motion": dict(cycle_motion=True),
           "use_mean_reset": dict(use_mean_reset=True), "discriminator": dict(disc=object()), "430 floats, the policy reads 934": dict(obs_size=934),
           "385 floats": dict(version=7), "358-float self observation": dict(vae_S=934), "69 dof": dict(dof=72), "latent has 64": dict(E=64),
           "acts in 69": dict(A=69)}
    for msg, kw in bad.items():
        with pytest.raises(PulseError, match=msg):
            ImZStepsB200(*_pieces(**kw), sim={})
    with pytest.raises(PulseError, match="tracked configuration"):
        ImZStepsB200(NS(track=object(), cfg=NS(cycle_motion=False, use_mean_reset=False), obs_size=430), *_pieces()[1:], sim={})
    sim = {k: torch.zeros(4) for k in SIM_KEYS}
    comp, pol, vae = _pieces()
    with pytest.raises(PulseError, match="dof_force"):                # power_reward is on by default
        ImZStepsB200(comp, pol, vae, sim=sim)
    for k in SIM_KEYS:
        with pytest.raises(PulseError, match=f"sim lacks \\['{k}'\\]"):
            ImZStepsB200(comp, pol, vae, sim=dict(sim, dof_force=torch.zeros(4), **{k: None}))


def _random_state(n, seed):
    g = torch.Generator().manual_seed(seed)
    q = lambda: torch.nn.functional.normalize(torch.randn(n, 24, 4, generator=g), dim=-1)
    v = lambda s: s * torch.randn(n, 24, 3, generator=g)
    body = dict(pos=v(0.5) + torch.tensor([0.0, 0.0, 0.9]), rot=q(), vel=v(1.0), ang=v(2.0))
    ref = dict(pos=body["pos"] + v(0.05), rot=q(), vel=v(1.0), ang=v(2.0))
    return body, ref


@pytest.mark.parametrize("ids", [TRACK_VR, (23, 5, 13, 0, 18), (7,), tuple(range(24))])
def test_track_columns_match_the_oracle(ids):
    """v6 and v7 of a body subset are column selections of the full-body v6 block: the map turns the oracle's full v6 row into its
    `imitation_obs_v6` / `imitation_obs_v7` of the subset bit for bit (elementwise fp32 expressions, no reduction across bodies)."""
    from oracle.pulse_oracle import imitation_obs_v6, imitation_obs_v7
    from pulse_b200.humanoid_im import track_columns
    n = 257
    b, r = _random_state(n, seed=len(ids))
    root_pos, root_rot = b["pos"][:, 0], b["rot"][:, 0]
    full = imitation_obs_v6(root_pos, root_rot, b["pos"], b["rot"], b["vel"], b["ang"], r["pos"], r["rot"], r["vel"], r["ang"])
    assert full.shape == (n, 576)
    sel = list(ids)
    sub = lambda d, k: d[k][:, sel]
    v6 = imitation_obs_v6(root_pos, root_rot, sub(b, "pos"), sub(b, "rot"), sub(b, "vel"), sub(b, "ang"), sub(r, "pos"), sub(r, "rot"),
                          sub(r, "vel"), sub(r, "ang"))
    v7 = imitation_obs_v7(root_pos, root_rot, sub(b, "pos"), sub(b, "vel"), sub(r, "pos"), sub(r, "vel"))
    assert torch.equal(full[:, track_columns(6, ids)], v6)
    assert torch.equal(full[:, track_columns(7, ids)], v7)
    if len(ids) == 24 and sel == sorted(sel):
        assert torch.equal(track_columns(6, ids), torch.arange(576))


def test_philox_blocks_never_repeat_across_steps_and_horizons():
    """Reset and latent draws over three horizons of 32 steps (the policy's offset moving on by 32 after each): no Philox block is
    read twice, and the keying is the one the header documents."""
    from pulse_b200.imz_rollout import philox_blocks
    T, n = 32, 3072
    seen, total = set(), 0
    for env in (0, 1, 777, n - 1):
        for h in range(3):
            for t in range(T):
                blocks = philox_blocks(env, t, h * T)
                total += len(blocks)
                seen.update(blocks)
    assert len(seen) == total
    b = philox_blocks(5, 3, 64)
    assert b[0] == ("reset", 5, 67) and b[1:] == [("policy", 5 * 64 + p, 67) for p in range(16)]


def _task(**kw):
    """A stand-in HumanoidImZ task: the attributes `compute_from_task` reads, with a MotionLibB200 that holds no tables."""
    from pulse_b200.motion_lib import MotionLibB200
    ml = MotionLibB200.__new__(MotionLibB200)
    ml._device = "cpu"
    t = NS(_motion_lib=ml, device="cpu", dt=1 / 30, reward_specs={"k_pos": 100.0, "k_rot": 10.0, "k_vel": 0.1, "k_ang_vel": 0.1, "w_pos": 0.5,
                                                                    "w_rot": 0.3, "w_vel": 0.1, "w_ang_vel": 0.1},
           power_reward=True, power_coefficient=0.0005, _reset_bodies_id=torch.tensor(TRACK_VR), _enable_early_termination=True, cycle_motion=False,
           max_episode_length=300, _termination_distances=torch.full((24,), 0.5), _track_bodies_id=torch.tensor([18, 23, 13]), obs_v=6)
    for k, v in kw.items():
        setattr(t, k, v)
    return t





def test_compute_from_task(lib):
    """The task's settings, its tracked bodies in the task's order and its observation version (4 maps to 6); every task setting under
    which the task's observation is not the tracked row is refused by name."""
    from pulse_b200 import PulseError
    from pulse_b200.imz_rollout import compute_from_task
    comp = compute_from_task(_task())
    assert tuple(comp.cfg.track_body_ids) == (18, 23, 13) and [comp.track.rank[j] for j in (18, 23, 13, 0)] == [0, 1, 2, -1]
    assert comp.cfg.obs_version == 6 and comp.obs_size == 430 and comp.reset_body_mask == (1 << 13) | (1 << 18) | (1 << 23)
    assert float(comp.termination_distances[0]) == 0.5 and comp.cfg.dt == float(torch.tensor(1 / 30, dtype=torch.float32))
    assert compute_from_task(_task(obs_v=4)).cfg.obs_version == 6
    assert compute_from_task(_task(obs_v=7)).obs_size == 358 + 27
    bad = {"obs_v 8": dict(obs_v=8), "fut_tracks": dict(_fut_tracks=True), "zero_out_far": dict(zero_out_far=True),
           "occlusion": dict(_occl_training=True), "full_body_reward False": dict(_full_body_reward=False), "self_obs_v 2": dict(self_obs_v=2),
           "observation noise": dict(add_obs_noise=True), "non-upright start": dict(_has_upright_start=False)}
    for msg, kw in bad.items():
        with pytest.raises(PulseError, match=msg):
            compute_from_task(_task(**kw))
