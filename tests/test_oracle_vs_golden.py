"""Pins oracle/pulse_oracle.py to the fixtures the reference produced (tests/golden/make_golden.py).

Integer outputs must be identical.  Float outputs are compared with atol 2e-6 (same PyTorch CPU
library and op order as the reference; the slack only covers reduction-order differences).
"""
import os

import numpy as np
import pytest
import torch

from oracle import pulse_oracle as po
from tests.helpers import load_npz, oracle_tables

ATOL = 2e-6


def close(a, b, atol=ATOL, rtol=1e-6):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    torch.testing.assert_close(a, b, atol=atol, rtol=rtol, equal_nan=True)


def test_quaternion_primitives():
    z = load_npz("quat.npz")
    close(po.slerp(z["qa"], z["qb"], z["t"]), z["slerp"])
    close(po.quat_mul(z["qa"], z["qb"]), z["quat_mul"])
    close(po.quat_rotate(z["qa"], z["qb"][:, :3]), z["rotate"])
    close(po.quat_to_exp_map(z["qe"]), z["exp_map"])
    ang, axis = po.quat_to_angle_axis(z["qe"])
    close(ang, z["angle"])
    close(axis, z["axis"])
    close(po.quat_to_six(z["qe"]), z["tan_norm"])
    close(po.heading_angle(z["qe"]), z["heading"])
    close(po.heading_quat(z["qe"]), z["heading_quat"])
    close(po.heading_quat(z["qe"], inverse=True), z["heading_quat_inv"])
    close(po.exp_map_to_quat(z["em"]), z["exp_map_to_quat"])


def test_motion_state_queries():
    tb = oracle_tables()
    z = load_npz("motion_state.npz")
    out = po.motion_state(tb, z["ids"], z["times"], z["offset"])
    assert torch.equal(out["frame_idx0"], z["frame_idx0"])
    assert torch.equal(out["frame_idx1"], z["frame_idx1"])
    assert torch.equal(out["blend"], z["blend"])
    for k in ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "motion_aa", "rg_pos", "rb_rot",
              "body_vel", "body_ang_vel"):
        close(out[k], z[k])
    close(po.root_pos_smpl(tb, z["ids"], z["times"]), z["root_pos_smpl"])
    assert torch.equal(po.sample_time_interval(tb, z["ids"], z["phase"]), z["sampled_time"])


@pytest.mark.parametrize("tag", ["n2", "n257"])
def test_humanoid_im_step(tag):
    tb = oracle_tables()
    z = load_npz(f"step_{tag}.npz")
    assert np.float32(z["dt"]) == np.float32(po.STEP_DT)
    out = po.humanoid_im_step(tb, po.ImStepConfig(), z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"],
                              z["motion_ids"], z["start_times"], z["start_offset"], z["global_offset"], z["cycle_counter"],
                              z["reset_buf_in"])
    assert torch.equal(out["frame_idx_rew"], z["frame_idx_rew"])
    assert torch.equal(out["frame_idx_obs"], z["frame_idx_obs"])
    assert torch.equal(out["reset_buf"], z["reset_buf"])
    assert torch.equal(out["terminate_buf"], z["terminate_buf"])
    assert out["reset_buf"].dtype == torch.int64
    close(out["rew_buf"], z["rew_buf"])
    close(out["reward_raw"], z["reward_raw"])
    close(out["obs_buf"], z["obs_buf"])
    close(out["obs_buf"][:, :po.SELF_OBS], z["self_obs"])
    close(out["ref_body_pos"], z["ref_body_pos"])
    close(out["ref_body_rot"], z["ref_body_rot"])
    close(out["ref_dof_pos"], z["ref_dof_pos"])
    # the fixture has terminations, time-outs and recovering envs in it
    if tag == "n257":
        assert 0 < int(z["terminate_buf"].sum()) < 257 and int(z["reset_buf"].sum()) > int(z["terminate_buf"].sum())


def test_mean_reset_and_v7_obs():
    tb = oracle_tables()
    z = load_npz("step_n257.npz")
    cfg = po.ImStepConfig(use_mean_reset=True, termination_distance=0.08)
    out = po.humanoid_im_step(tb, cfg, z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"],
                              z["start_times"], z["start_offset"], z["global_offset"], torch.zeros_like(z["cycle_counter"]),
                              z["reset_buf_in"])
    assert torch.equal(out["reset_buf"], z["reset_buf_mean"])
    assert torch.equal(out["terminate_buf"], z["terminate_buf_mean"])
    bs = z["body_state"]
    track = [13, 18, 23]
    t_obs = po.im_motion_times(z["progress_buf"], z["start_times"], z["start_offset"], po.STEP_DT, True)
    nxt = po.motion_state(tb, z["motion_ids"], t_obs, z["global_offset"])
    v7 = po.imitation_obs_v7(bs[:, 0, 0:3], bs[:, 0, 3:7], bs[:, track, 0:3], bs[:, track, 7:10],
                             nxt["rg_pos"][:, track], nxt["body_vel"][:, track])
    close(v7, z["task_obs_v7"])


def test_amp_observation():
    z = load_npz("step_n257.npz")
    bs = z["body_state"]
    cur = po.amp_obs_smpl(bs[:, 0, 0:3], bs[:, 0, 3:7], bs[:, 0, 7:10], bs[:, 0, 10:13], z["dof_pos"], z["dof_vel"],
                          bs[:, list(po.KEY_BODY_IDS), 0:3], po.amp_dof_subset())
    assert cur.shape[1] == po.AMP_OBS
    close(cur, z["amp_cur"])
    nh = z["amp_hist_in"].shape[0]
    new = po.amp_obs_step(z["amp_hist_in"], bs[:nh], z["dof_pos"][:nh], z["dof_vel"][:nh])
    close(new, z["amp_hist_out"])


def test_agent_arithmetic():
    z = load_npz("agent.npz")
    advs = po.discount_values(z["fdones"], z["values"], z["rewards"], z["next_values"])
    close(advs, z["advs"])
    close(advs + z["values"], z["returns"])
    adv_norm = po.normalized_advantages(po.swap_and_flatten01(z["returns"]), po.swap_and_flatten01(z["values"]))
    close(adv_norm, z["adv_norm"])
    close(po.actor_loss(z["old_neglogp"], z["new_neglogp"], z["adv_b"]), z["actor_loss"])
    close(po.critic_loss(z["critic_values"], z["critic_returns"]), z["critic_loss"])
    close(po.bound_loss(z["mu"]), z["bound_loss"])
    close(po.disc_reward(z["disc_logits"]), z["disc_reward"])
    close(po.kl_multi(z["kl_qm"], z["kl_qv"], z["kl_pm"], z["kl_pv"]), z["kl_multi"])
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    close(bce(z["disc_logits"], torch.zeros_like(z["disc_logits"])), z["bce_neg"])
    close(bce(z["disc_logits"], torch.ones_like(z["disc_logits"])), z["bce_pos"])
    # discriminator loss incl. gradient penalty, and its parameter gradients through autograd
    lin = lambda w, b: (lambda x: torch.nn.functional.linear(x, w, b))
    ws = [z[k].clone().requires_grad_(True) for k in ("disc_w0", "disc_b0", "disc_w1", "disc_b1", "disc_w2", "disc_b2")]
    dmlp = lambda x: lin(ws[4], ws[5])(torch.relu(lin(ws[2], ws[3])(torch.relu(lin(ws[0], ws[1])(x)))))
    dinfo = po.disc_loss(dmlp, z["disc_agent"], z["disc_replay"], z["disc_demo"], ws[4], [ws[0], ws[2], ws[4]])
    close(dinfo["disc_loss"], z["disc_loss"])
    close(dinfo["disc_grad_penalty"], z["disc_grad_penalty"])
    close(dinfo["disc_agent_acc"], z["disc_agent_acc"])
    close(dinfo["disc_demo_acc"], z["disc_demo_acc"])
    grads = torch.autograd.grad(dinfo["disc_loss"], ws)
    for g_, k in zip(grads, ("disc_gw0", "disc_gb0", "disc_gw1", "disc_gb1", "disc_gw2", "disc_gb2")):
        close(g_, z[k], atol=1e-5)
    rms = po.RunningMeanStd(7)
    y1 = rms.normalize(z["rms_x1"]); rms.update(z["rms_x1"])
    y2 = rms.normalize(z["rms_x2"]); rms.update(z["rms_x2"])
    y3 = rms.normalize(z["rms_x1"])
    close(y1, z["rms_y1"]); close(y2, z["rms_y2"]); close(y3, z["rms_y3"])
    torch.testing.assert_close(rms.mean, z["rms_mean"], atol=1e-12, rtol=1e-12)
    torch.testing.assert_close(rms.var, z["rms_var"], atol=1e-12, rtol=1e-12)
    assert float(rms.count) == float(z["rms_count"])


def test_oracle_against_reference_pins():
    """The oracle against the reference's own functions on fresh seeded inputs (tests/golden/reference_pins.npz,
    make_golden_reference_pins.py: every 8th observation / reward row, every 4th slerp row)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_reference_pins", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                                                                              "make_golden_reference_pins.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    g = load_npz("reference_pins.npz")
    z, chk = m.pin_inputs()
    assert abs(chk - float(g["checksum"])) < 1e-9 * abs(chk)
    pos, rot, vel, ang, rpos, rrot, rvel, rang = (z[k] for k in ("pos", "rot", "vel", "ang", "rpos", "rrot", "rvel", "rang"))
    close(po.self_obs_smpl_max(pos, rot, vel, ang)[m.ROWS], g["self_obs"])
    close(po.imitation_obs_v6(pos[:, 0], rot[:, 0], pos, rot, vel, ang, rpos, rrot, rvel, rang)[m.ROWS], g["imitation_obs_v6"])
    r2, raw2 = po.imitation_reward(pos, rot, vel, ang, rpos, rrot, rvel, rang)
    close(r2[m.ROWS], g["reward"]); close(raw2[m.ROWS], g["reward_raw"])
    close(po.slerp(z["q0"], z["q1"], z["t"])[m.SLERP_ROWS], g["slerp"])


def test_vae_distillation_teacher_zdecode_reach_pd():
    """SURVEY rows a14 / a19 / a20: the oracle's restatement of AMPZBuilder.Network + _optimize_kin, the PNN teacher,
    HumanoidZ.compute_z_actions, the reach task functions and the PD target map against reference-generated vectors."""
    from tests.helpers import vae_golden, vae_param_list
    g, _, nets, d, pnn_cols, composer = vae_golden()
    params = vae_param_list(nets)
    for tag, regu in (("", False), ("regu_", True)):
        for p in params.values():
            p.requires_grad_(True)
            p.grad = None
        r = po.vae_kin_loss(nets, g["obs"], g[tag + "noise"], g["gt_action"], g["progress"], d["T"], use_regu=regu)
        r["kin_loss"].backward()
        for k in ("kin_loss", "kin_action_loss", "kin_KLD", "kin_ar1"):
            close(r[k].detach(), torch.as_tensor(g[tag + "info." + k]))
        if regu:
            close(r["kin_prior_regu"].detach(), torch.as_tensor(g["regu_info.kin_prior_regu"]))
        for name, p in params.items():
            close(p.grad, g[tag + "grad." + name], atol=1e-6, rtol=1e-5)
    with torch.no_grad():
        for k in ("pred_action", "vae_mu", "vae_log_var", "prior_mu", "prior_log_var"):
            close(r[k], g[k])
        assert float((g["vae_log_var"] >= 2).float().mean()) > 0.05      # the clamp is exercised
        close(po.vae_eval_critic(nets, g["obs"]), g["value"])
        ta, w = po.teacher_action(g["teacher_raw_obs"], g["teacher_mean"], g["teacher_var"], pnn_cols, composer, d["S"])
        close(ta, g["teacher_action"]); close(w, g["teacher_weights"])
        close(po.z_decode_actions(nets, g["teacher_raw_obs"], g["teacher_mean"], g["teacher_var"], g["action_z"]), g["z_actions"])
        close(po.reach_obs(g["reach_root_states"], g["reach_tar_pos"]), g["reach_obs"])
        close(po.reach_reward(g["reach_body_pos"], g["reach_tar_pos"]), g["reach_reward"])
        close(po.pd_targets(g["gt_action"], g["pd_offset"], g["pd_scale"]), g["pd_target"])
    assert abs(po.kld_anneal(3750) - 0.0055) < 1e-9 and po.kld_anneal(6000) == 0.001


def _check_against_step4096(out, g, obs_atol, sum_atol):
    assert torch.equal(out["reset_buf"], g["reset_buf"]) and torch.equal(out["terminate_buf"], g["terminate_buf"])
    assert torch.equal(out["frame_idx_rew"], g["frame_idx_rew"]) and torch.equal(out["frame_idx_obs"], g["frame_idx_obs"])
    close(out["rew_buf"], g["rew_buf"], atol=obs_atol, rtol=0)
    close(out["reward_raw"], g["reward_raw"], atol=obs_atol, rtol=0)
    close(out["obs_buf"][::32], g["obs_rows"], atol=obs_atol, rtol=0)
    close(out["obs_buf"].double().sum(1), g["obs_row_sum"], atol=sum_atol, rtol=0)


def test_step_4096_envs_oracle_matches_reference():
    """BASELINE config C2 size (4096 envs, 100 clips): the oracle's fused step on the regenerated inputs vs the reference's outputs
    (tests/golden/step_n4096.npz, make_golden_step4096.py); also proves the bit-exact input regeneration on this host."""
    from tests.helpers import exact_step_inputs, exact_tables, load_npz as _l
    g = _l("step_n4096.npz")
    tb = exact_tables(int(g["dims"][1]))
    z, chk = exact_step_inputs(tb, int(g["dims"][0]))
    assert abs(chk - float(g["checksum"])) < 1e-9 * abs(chk)
    out = po.humanoid_im_step(tb, po.ImStepConfig(), z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"],
                              z["start_times"], z["start_offset"], z["global_offset"], z["cycle_counter"], z["reset_buf_in"])
    _check_against_step4096(out, g, 2e-6, 1e-4)
    assert 0 < int(g["terminate_buf"].sum()) < 4096 and int(g["reset_buf"].sum()) > int(g["terminate_buf"].sum())


def test_vae_full_width_oracle_matches_reference():
    """Row a19 at im_z_fit.yaml widths: the oracle on the regenerated fixture vs the reference's losses / gradient samples
    (tests/golden/vae_full.npz).  Also proves the integer-exact fixture regeneration (checksum) on this host."""
    from tests.helpers import VAE_FULL, load_npz as _l, vae_full_fixture, vae_param_list
    g = _l("vae_full.npz")
    sd, batch, chk = vae_full_fixture()
    assert abs(chk - float(g["checksum"])) < 1e-9 * max(1.0, abs(chk))
    nets = po.VaeNets.from_state_dict(sd, VAE_FULL["S"])
    params = vae_param_list(nets)
    for p in params.values():
        p.requires_grad_(True)
    r = po.vae_kin_loss(nets, batch["obs"], batch["noise"], batch["gt_action"], batch["progress"], VAE_FULL["T"])
    r["kin_loss"].backward()
    for k in ("kin_loss", "kin_action_loss", "kin_KLD", "kin_ar1"):
        close(r[k].detach(), torch.as_tensor(g["info." + k]), atol=1e-5, rtol=1e-5)
    for name, p in params.items():
        ref = g["grad." + name]
        close(p.grad[:4] if p.grad.dim() == 2 else p.grad, ref, atol=2e-6, rtol=1e-3)
    with torch.no_grad():
        for k in ("pred_action", "vae_mu", "vae_log_var", "prior_mu", "prior_log_var"):
            close(r[k][:64], g[k], atol=2e-5, rtol=1e-4)
    assert float((g["vae_log_var"] >= 2).float().mean()) > 0.02      # the clamp is exercised at full width too


def test_reach_full_step_pieces():
    from tests.helpers import load_npz as _l
    g = _l("vae.npz")
    bs = g["reach_body_state"]
    rs, tm = po.humanoid_reset(g["reach_progress"], g["reach_contact"], g["reach_contact_ids"], bs[..., 0:3], 300, True, g["reach_term_h"])
    assert torch.equal(rs, g["reach_reset"]) and torch.equal(tm, g["reach_terminate"])
    assert 0 < int(tm.sum()) < tm.numel()
    close(po.self_obs_smpl_max(bs[..., 0:3], bs[..., 3:7], bs[..., 7:10], bs[..., 10:13]), g["reach_self_obs"])
    close(po.reach_obs(bs[:, 0, :], g["reach_tar_pos"]), g["reach_obs_full"])
    close(po.reach_reward(bs[:, 23, 0:3], g["reach_tar_pos"]), g["reach_reward_full"])


def test_motionlib_loader_per_clip_pipeline():
    """SURVEY 8(f)-1 groundwork: the oracle's restatement of the per-clip loader (heading randomisation, local rotations, forward
    kinematics, gaussian-filtered velocities, dof velocities) reproduces the reference's tables EXACTLY, including its mix of
    float64 / float32 stages (tests/golden/loader.npz, make_golden_loader.py; the same rows as motionlib.npz)."""
    from tests.helpers import load_npz as _l
    z = _l("loader.npz")
    tables = _l("motionlib.npz")
    nf = z["num_frames"].tolist()
    start = 0
    for i, n in enumerate(nf):
        a, b = start, start + n
        start = b
        _, q, tr = po.loader_heading(z["in_pose_aa"][a:b], z["in_pose_quat_global"][a:b].numpy(), z["in_root_trans"][a:b], float(z["headings"][i]))
        out = po.loader_clip(q, tr, float(z["fps"][i]), z["parents"].tolist(), z["local_translation"])
        for k, v in out.items():
            assert torch.equal(v.double(), z[k][a:b]), (i, k)
            assert torch.equal(v.float(), tables[k][a:b]), (i, k)      # what load_motions() concatenates (fp32)
