"""GPU parity tests of the step path: CUDA kernels (through the C ABI) vs golden fixtures / oracle.

Bars (BASELINE.json north_star): frame indices and reset/terminate masks bit-exact; observations
and rewards within 1e-4.
"""
import pytest
import torch

from tests.helpers import load_npz, oracle_tables, synthetic_step_inputs, synthetic_tables

pytestmark = pytest.mark.gpu
OBS_ATOL = 1e-4


def _dev():
    return torch.device("cuda:0")


def _tables_to_dict(tb):
    return {"gts": tb.gts, "grs": tb.grs, "lrs": tb.lrs, "gvs": tb.gvs, "gavs": tb.gavs, "dvs": tb.dvs, "motion_aa": tb.motion_aa,
            "lengths": tb.lengths, "num_frames": tb.num_frames, "dt": tb.dt, "length_starts": tb.length_starts, "fps": tb.fps,
            "motion_bodies": tb.motion_bodies, "motion_limb_weights": tb.motion_limb_weights}


def _mlib(tb):
    from pulse_b200.motion_lib import MotionLibB200
    return MotionLibB200.from_tables(_tables_to_dict(tb), device=_dev())


def _run_step(ml, z, cfg=None, bodies_per_env=24, obs_stride=934, flags=7, env_ids=None, dof_interleaved=True, with_ref=True):
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    dev = _dev()
    n = z["body_state"].shape[0]
    comp = HumanoidImCompute(ml, cfg or ImConfig())
    full = torch.full((n, bodies_per_env, 13), 7.0, device=dev)
    full[:, :24] = z["body_state"].to(dev)
    dof_state = torch.zeros(n, 69 + (3 if dof_interleaved else 0), 2, device=dev)
    dof_state[:, :69, 1] = z["dof_vel"].to(dev)
    dof_vel = dof_state[:, :69, 1] if dof_interleaved else z["dof_vel"].to(dev).contiguous()
    out = {
        "obs_buf": torch.full((n, obs_stride), -9.0, device=dev), "self_obs_buf": torch.zeros(n, 358, device=dev),
        "rew_buf": torch.zeros(n, device=dev), "reward_raw": torch.zeros(n, 5, device=dev),
        "reset_buf": torch.full((n,), -1, dtype=torch.long, device=dev), "terminate_buf": torch.full((n,), -1, dtype=torch.long, device=dev),
        "pass_time": torch.zeros(n, dtype=torch.uint8, device=dev),
    }
    if with_ref:
        out.update(ref_body_pos=torch.zeros(n, 24, 3, device=dev), ref_body_vel=torch.zeros(n, 24, 3, device=dev),
                   ref_body_rot=torch.zeros(n, 24, 4, device=dev), ref_dof_pos=torch.zeros(n, 69, device=dev))
    comp.step(body_state=full, dof_vel=dof_vel, dof_force=z["dof_force"].to(dev), progress_buf=z["progress_buf"].to(dev),
              motion_ids=z["motion_ids"].to(dev), motion_start_times=z["start_times"].to(dev), motion_start_offset=z["start_offset"].to(dev),
              global_offset=z["global_offset"].to(dev), cycle_counter=z["cycle_counter"].to(dev), env_ids=env_ids, flags=flags, **out)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def _check_step(out, ref, n_obs=934):
    assert torch.equal(out["reset_buf"], ref["reset_buf"])
    assert torch.equal(out["terminate_buf"], ref["terminate_buf"])
    torch.testing.assert_close(out["rew_buf"], ref["rew_buf"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(out["reward_raw"], ref["reward_raw"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(out["obs_buf"][:, :n_obs], ref["obs_buf"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(out["self_obs_buf"], ref["obs_buf"][:, :358], atol=OBS_ATOL, rtol=0)
    if "ref_body_pos" in out:
        torch.testing.assert_close(out["ref_body_pos"], ref["ref_body_pos"], atol=1e-5, rtol=0)
        torch.testing.assert_close(out["ref_body_rot"], ref["ref_body_rot"], atol=OBS_ATOL, rtol=0)
        torch.testing.assert_close(out["ref_body_vel"], ref["ref_body_vel"], atol=1e-5, rtol=0)
        # exponential maps reach pi in magnitude and inherit the conditioning of the reference's slerp (theta from acos(dot), sin(theta) from
        # sqrt(1 - dot^2)): one ulp in the dot product moves |q| by 6e-8 / theta^2, so this side buffer is compared relative + absolute
        torch.testing.assert_close(out["ref_dof_pos"], ref["ref_dof_pos"], atol=OBS_ATOL, rtol=1e-4)


def test_motion_state_matches_reference_golden():
    ml = _mlib(oracle_tables())
    z = load_npz("motion_state.npz")
    dev = _dev()
    out = ml.get_motion_state(z["ids"].to(dev), z["times"].to(dev), z["offset"].to(dev), diagnostics=True)
    torch.cuda.synchronize()
    assert torch.equal(out["frame_idx0"].cpu(), z["frame_idx0"])
    assert torch.equal(out["frame_idx1"].cpu(), z["frame_idx1"])
    assert torch.equal(out["blend"].cpu(), z["blend"])
    for k in ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "motion_aa", "rg_pos", "rb_rot", "body_vel",
              "body_ang_vel"):
        # rotations go through slerp (acos / sin of tiny angles): the 1e-4 observation bar applies
        tol = 1e-4 if k in ("root_rot", "rb_rot", "dof_pos") else 1e-5
        torch.testing.assert_close(out[k].cpu(), z[k], atol=tol, rtol=0, msg=lambda m, k=k: f"{k}: {m}")
    rp = ml.get_root_pos_smpl(z["ids"].to(dev), z["times"].to(dev))["root_pos"].cpu()
    torch.testing.assert_close(rp, z["root_pos_smpl"], atol=1e-6, rtol=0)
    st = ml.sample_time_interval(z["ids"].to(dev), phase=z["phase"].to(dev)).cpu()
    assert torch.equal(st, z["sampled_time"])
    empty = ml.get_motion_state(z["ids"][:0].to(dev), z["times"][:0].to(dev))
    assert empty["rg_pos"].shape == (0, 24, 3)


@pytest.mark.parametrize("tag", ["n2", "n257"])
def test_im_step_matches_reference_golden(tag):
    ml = _mlib(oracle_tables())
    z = load_npz(f"step_{tag}.npz")
    out = _run_step(ml, z)
    _check_step(out, z)


def test_im_step_mean_reset_matches_reference_golden():
    from pulse_b200.humanoid_im import ImConfig
    ml = _mlib(oracle_tables())
    z = load_npz("step_n257.npz")
    z = dict(z)
    z["cycle_counter"] = torch.zeros_like(z["cycle_counter"])
    out = _run_step(ml, z, cfg=ImConfig(use_mean_reset=True, termination_distance=0.08))
    assert torch.equal(out["reset_buf"], z["reset_buf_mean"])
    assert torch.equal(out["terminate_buf"], z["terminate_buf_mean"])


MIXED_RATES = (24.0, 25.0, 29.97, 30.0, 50.0, 60.0, 120.0)


@pytest.mark.parametrize("n_envs,n_motions,fps", [pytest.param(1, 3, 30.0, id="1-3"), pytest.param(4099, 300, 30.0, id="4099-300"),
                                                  pytest.param(4099, 300, MIXED_RATES, id="4099-300-mixed-fps")])
def test_im_step_matches_oracle_random(n_envs, n_motions, fps):
    """Mixed rates: above 30 fps the observation time runs more than a frame ahead of the reward time, so the reward and observation
    queries can need four distinct frame rows; the fourth has no copy slot and is read straight from the records (im_step.cu's planner)."""
    from oracle import pulse_oracle as po
    tb = synthetic_tables(n_motions, seed=3, max_frames=200, median_frames=60, fps=fps)
    z = synthetic_step_inputs(tb, n_envs, seed=5)
    ref = po.humanoid_im_step(tb, po.ImStepConfig(), z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"],
                              z["start_times"], z["start_offset"], z["global_offset"], z["cycle_counter"], z["reset_buf_in"])
    out = _run_step(_mlib(tb), z)
    _check_step(out, ref)
    assert 0 < int(ref["terminate_buf"].sum()) < n_envs or n_envs == 1
    rows = torch.cat([ref["frame_idx_rew"], ref["frame_idx_obs"]], 1)
    four = int(sum(len(set(r)) == 4 for r in rows.tolist()))
    print(f"\n{four} of {n_envs} envs need four distinct frame rows")
    if fps != 30.0:
        assert four > 0


def test_im_step_strided_unaligned_views():
    """Isaac Gym views: bodies_per_env > 24 (rows only 4-byte aligned), obs rows with a stride."""
    ml = _mlib(oracle_tables())
    z = load_npz("step_n257.npz")
    out = _run_step(ml, z, bodies_per_env=25, obs_stride=941, dof_interleaved=True)
    _check_step(out, z)
    assert torch.all(out["obs_buf"][:, 934:] == -9.0)  # nothing written past the row
    out2 = _run_step(ml, z, bodies_per_env=27, obs_stride=936, dof_interleaved=False, with_ref=False)
    _check_step(out2, z)


def test_im_step_staged_flags_and_env_subset():
    from pulse_b200 import _lib
    ml = _mlib(oracle_tables())
    z = load_npz("step_n257.npz")
    o1 = _run_step(ml, z, flags=_lib.STEP_REWARD)
    torch.testing.assert_close(o1["rew_buf"], z["rew_buf"], atol=OBS_ATOL, rtol=0)
    assert torch.all(o1["reset_buf"] == -1) and torch.all(o1["obs_buf"] == -9.0)
    o2 = _run_step(ml, z, flags=_lib.STEP_RESET | _lib.STEP_OBS)
    assert torch.equal(o2["reset_buf"], z["reset_buf"]) and torch.equal(o2["terminate_buf"], z["terminate_buf"])
    torch.testing.assert_close(o2["obs_buf"], z["obs_buf"], atol=OBS_ATOL, rtol=0)
    # pass_time mask == (t >= motion_len)
    from oracle import pulse_oracle as po
    tb = oracle_tables()
    t = po.im_motion_times(z["progress_buf"], z["start_times"], z["start_offset"], po.STEP_DT, False)
    assert torch.equal(o2["pass_time"].bool(), t >= tb.lengths[z["motion_ids"]])
    ids = torch.tensor([5, 0, 200, 17, 256], dtype=torch.long, device=_dev())
    o3 = _run_step(ml, z, flags=_lib.STEP_OBS, env_ids=ids)
    sel = ids.cpu()
    torch.testing.assert_close(o3["obs_buf"][sel], z["obs_buf"][sel], atol=OBS_ATOL, rtol=0)
    mask = torch.ones(257, dtype=torch.bool)
    mask[sel] = False
    assert torch.all(o3["obs_buf"][mask] == -9.0)


def test_im_step_rejects_bad_arguments():
    from pulse_b200 import PulseError
    from pulse_b200.humanoid_im import HumanoidImCompute
    ml = _mlib(oracle_tables())
    z = load_npz("step_n2.npz")
    comp = HumanoidImCompute(ml)
    dev = _dev()
    kw = dict(body_state=z["body_state"].to(dev), progress_buf=z["progress_buf"].to(dev), motion_ids=z["motion_ids"].to(dev),
              motion_start_times=z["start_times"].to(dev), motion_start_offset=z["start_offset"].to(dev), global_offset=z["global_offset"].to(dev))
    with pytest.raises(PulseError):
        comp.step(flags=4, obs_buf=torch.zeros(2, 900, device=dev), **kw)
    with pytest.raises(PulseError):
        comp.step(flags=4, obs_buf=torch.zeros(2, 934, device=dev), **{**kw, "progress_buf": z["progress_buf"].to(dev).int()})
    with pytest.raises(PulseError):
        comp.step(flags=8, obs_buf=torch.zeros(2, 934, device=dev), **kw)


def test_amp_obs_matches_reference_golden():
    from pulse_b200.humanoid_im import HumanoidImCompute
    ml = _mlib(oracle_tables())
    comp = HumanoidImCompute(ml)
    z = load_npz("step_n257.npz")
    dev = _dev()
    nh = z["amp_hist_in"].shape[0]
    dof_state = torch.zeros(257, 72, 2, device=dev)
    dof_state[:, :69, 0] = z["dof_pos"].to(dev)
    dof_state[:, :69, 1] = z["dof_vel"].to(dev)
    body = torch.zeros(257, 26, 13, device=dev)
    body[:, :24] = z["body_state"].to(dev)
    buf = torch.zeros(257, 10, 196, device=dev)
    buf[:nh] = z["amp_hist_in"].to(dev)
    comp.amp_obs(body_state=body, dof_pos=dof_state[:, :69, 0], dof_vel=dof_state[:, :69, 1], amp_obs_buf=buf)
    torch.cuda.synchronize()
    torch.testing.assert_close(buf[:, 0].cpu(), z["amp_cur"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(buf[:nh].cpu(), z["amp_hist_out"], atol=OBS_ATOL, rtol=0)
    assert torch.equal(buf[:nh, 1:].cpu(), z["amp_hist_in"][:, :9])  # history moved bit-exactly
    buf2 = buf.clone()
    comp.amp_obs(body_state=body, dof_pos=dof_state[:, :69, 0], dof_vel=dof_state[:, :69, 1], amp_obs_buf=buf2, shift_history=False)
    torch.cuda.synchronize()
    assert torch.equal(buf2, buf)


def test_full_size_properties():
    """BASELINE config C4 size (16384 envs): size-independent invariants of the fused step.

    (1) yaw invariance: rotating the whole world (sim state, motion tables, offsets) about z leaves
        observations and rewards unchanged;  (2) a humanoid exactly on the reference pose gets the full
        imitation reward and zero difference blocks;  (3) linear index check on frame indices."""
    from oracle import pulse_oracle as po
    n = 16384
    tb = synthetic_tables(1024, seed=11, max_frames=300, median_frames=120)
    z = synthetic_step_inputs(tb, n, seed=13)
    z["global_offset"] = torch.zeros_like(z["global_offset"])
    base = _run_step(_mlib(tb), z, with_ref=False)
    # (1) rotate everything by yaw
    ang = torch.tensor(0.7)
    qz = torch.tensor([0.0, 0.0, torch.sin(ang / 2), torch.cos(ang / 2)])
    rot_v = lambda v: po.quat_rotate(qz.expand(*v.shape[:-1], 4), v)
    rot_q = lambda q: po.quat_mul(qz.expand_as(q), q)
    import dataclasses
    tb2 = dataclasses.replace(tb, gts=rot_v(tb.gts), grs=rot_q(tb.grs), gvs=rot_v(tb.gvs), gavs=rot_v(tb.gavs))
    z2 = dict(z)
    bs = z["body_state"]
    z2["body_state"] = torch.cat([rot_v(bs[..., 0:3]), rot_q(bs[..., 3:7]), rot_v(bs[..., 7:10]), rot_v(bs[..., 10:13])], dim=-1)
    rot = _run_step(_mlib(tb2), z2, with_ref=False)
    torch.testing.assert_close(rot["obs_buf"], base["obs_buf"], atol=2e-4, rtol=0)
    torch.testing.assert_close(rot["rew_buf"], base["rew_buf"], atol=1e-4, rtol=0)
    assert (rot["reset_buf"] != base["reset_buf"]).float().mean() < 1e-3  # knife-edge flips only
    # (2) on-pose humanoid at t (reward) -- use obs time for the diff blocks
    t_rew = po.im_motion_times(z["progress_buf"], z["start_times"], z["start_offset"], po.STEP_DT, False)
    pose = po.motion_state(tb, z["motion_ids"], t_rew, None)
    z3 = dict(z)
    z3["body_state"] = torch.cat([pose["rg_pos"], torch.nn.functional.normalize(pose["rb_rot"], dim=-1), pose["body_vel"], pose["body_ang_vel"]], -1)
    z3["dof_force"] = torch.zeros_like(z["dof_force"])
    on = _run_step(_mlib(tb), z3, with_ref=False)
    assert torch.all(on["rew_buf"] > 0.97)
    assert int(on["terminate_buf"].sum()) == 0
    # (3) frame rows stay inside each clip: obs of an env never depends on another clip's frames ->
    # run the same env range twice with permuted env order and compare
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
    zp = {k: (v[perm] if torch.is_tensor(v) and v.shape[:1] == (n,) else v) for k, v in z.items()}
    pr = _run_step(_mlib(tb), zp, with_ref=False)
    assert torch.equal(pr["obs_buf"], base["obs_buf"][perm])
    assert torch.equal(pr["reset_buf"], base["reset_buf"][perm])


def _exact_case(n, clips):
    from tests.helpers import exact_step_inputs, exact_tables
    tb = exact_tables(clips)
    z, chk = exact_step_inputs(tb, n)
    return tb, z, chk


def test_step_4096_envs_matches_reference_golden():
    """BASELINE config C2 size: 4096 envs on 100 clips against the UNMODIFIED reference's outputs (tests/golden/step_n4096.npz)."""
    g = load_npz("step_n4096.npz")
    n, clips = int(g["dims"][0]), int(g["dims"][1])
    tb, z, chk = _exact_case(n, clips)
    assert abs(chk - float(g["checksum"])) < 1e-9 * abs(chk), "regenerated inputs differ from the ones the golden was made with"
    out = _run_step(_mlib(tb), z, with_ref=False)
    assert torch.equal(out["reset_buf"], g["reset_buf"]) and torch.equal(out["terminate_buf"], g["terminate_buf"])
    torch.testing.assert_close(out["rew_buf"], g["rew_buf"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(out["reward_raw"], g["reward_raw"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(out["obs_buf"][::32], g["obs_rows"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(out["obs_buf"].double().sum(1), g["obs_row_sum"], atol=934 * 2e-6, rtol=0)
    # frame indices through the MotionLib query entry (same planner arithmetic as the fused kernel)
    from oracle import pulse_oracle as po
    dev = _dev()
    ml = _mlib(tb)
    for plus, key in ((False, "frame_idx_rew"), (True, "frame_idx_obs")):
        t = po.im_motion_times(z["progress_buf"], z["start_times"], z["start_offset"], po.STEP_DT, plus)
        ms = ml.get_motion_state(z["motion_ids"].to(dev), t.to(dev), z["global_offset"].to(dev), diagnostics=True)
        assert torch.equal(torch.stack([ms["frame_idx0"], ms["frame_idx1"]], -1).cpu(), g[key])


def test_step_16384_envs_matches_oracle():
    """BASELINE config C4 size (the headline): all 16384 envs compared DIRECTLY with the oracle (bit-exact masks, 1e-4 floats)."""
    from oracle import pulse_oracle as po
    tb, z, _ = _exact_case(16384, 2048)
    ref = po.humanoid_im_step(tb, po.ImStepConfig(), z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"],
                              z["start_times"], z["start_offset"], z["global_offset"], z["cycle_counter"], z["reset_buf_in"])
    out = _run_step(_mlib(tb), z)
    _check_step(out, ref)
    assert 0 < int(ref["terminate_buf"].sum()) < 16384


def test_getup_recovery_masking_matches_oracle():
    """HumanoidImGetup._compute_reset (humanoid_im_getup.py:203-210) inside the fused kernel: recovering envs are never reset, their
    progress counter is pulled back by one and their observation is taken at that earlier time."""
    from oracle import pulse_oracle as po
    from pulse_b200.humanoid_im import HumanoidImCompute
    tb, z, _ = _exact_case(515, 40)
    g = torch.Generator().manual_seed(4)
    rec = (torch.rand(515, generator=g) < 0.3).int() * torch.randint(1, 150, (515,), generator=g, dtype=torch.int32)
    ref = po.humanoid_im_step(tb, po.ImStepConfig(), z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"],
                              z["start_times"], z["start_offset"], z["global_offset"], z["cycle_counter"], z["reset_buf_in"], recovery_counter=rec)
    dev = _dev()
    comp = HumanoidImCompute(_mlib(tb))
    n = 515
    prog = z["progress_buf"].to(dev).clone()
    out = {"obs_buf": torch.zeros(n, 934, device=dev), "rew_buf": torch.zeros(n, device=dev), "reward_raw": torch.zeros(n, 5, device=dev),
           "reset_buf": torch.full((n,), -1, dtype=torch.long, device=dev), "terminate_buf": torch.full((n,), -1, dtype=torch.long, device=dev)}
    fd = torch.full((n,), -1.0, device=dev)
    comp.step(body_state=z["body_state"].to(dev), dof_vel=z["dof_vel"].to(dev), dof_force=z["dof_force"].to(dev), progress_buf=prog,
              motion_ids=z["motion_ids"].to(dev), motion_start_times=z["start_times"].to(dev), motion_start_offset=z["start_offset"].to(dev),
              global_offset=z["global_offset"].to(dev), cycle_counter=z["cycle_counter"].to(dev), recovery_counter=rec.to(dev), fdones_out=fd, **out)
    torch.cuda.synchronize()
    assert torch.equal(prog.cpu(), ref["progress_buf"]) and int((prog.cpu() != z["progress_buf"]).sum()) == int((rec > 0).sum())
    assert torch.equal(out["reset_buf"].cpu(), ref["reset_buf"]) and torch.equal(out["terminate_buf"].cpu(), ref["terminate_buf"])
    assert torch.equal(fd.cpu(), ref["reset_buf"].float())
    assert int(ref["reset_buf"][rec > 0].sum()) == 0
    torch.testing.assert_close(out["obs_buf"].cpu(), ref["obs_buf"], atol=OBS_ATOL, rtol=0)
    torch.testing.assert_close(out["rew_buf"].cpu(), ref["rew_buf"], atol=OBS_ATOL, rtol=0)


def test_build_amp_obs_demo_matches_oracle():
    """humanoid_amp.py:253-284: demo AMP observations from the reference motion (MotionLib query + AMP obs)."""
    from oracle import pulse_oracle as po
    from pulse_b200.humanoid_im import HumanoidImCompute
    tb = oracle_tables()
    comp = HumanoidImCompute(_mlib(tb))
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, tb.num_motions, (37,), generator=g)
    t0 = po.sample_time_interval(tb, ids, torch.rand(37, generator=g))
    out = comp.build_amp_obs_demo(ids.to(_dev()), t0.to(_dev())).cpu()
    steps = 10
    rid = ids.unsqueeze(-1).repeat(1, steps).reshape(-1)
    rt = (t0.unsqueeze(-1) + (-po.STEP_DT) * torch.arange(0, steps)).reshape(-1)
    ms = po.motion_state(tb, rid, rt, None)
    ref = po.amp_obs_smpl(ms["root_pos"], ms["root_rot"], ms["root_vel"], ms["root_ang_vel"], ms["dof_pos"], ms["dof_vel"],
                          ms["rg_pos"][:, list(po.KEY_BODY_IDS)], po.amp_dof_subset()).view(37, steps * 196)
    torch.testing.assert_close(out, ref, atol=OBS_ATOL, rtol=0)
