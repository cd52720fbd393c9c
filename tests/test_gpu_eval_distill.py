"""The evaluation pass of the distillation student (`EvalStepsB200` over `DistillStepsB200`: the PULSE VAE at im_z_fit.yaml's widths,
z = the posterior mean, the decoder's action, no teacher) on the synthetic MotionLib and the device-side stand-in physics of
test_gpu_eval_pass.py, the displacement driven by the student's PD targets.

Bars: exact tracking gives zero metrics, no termination and success rate 1; the recorded frames fed to oracle/eval_oracle.py give the
same failed / success keys, step counts and `eval_info` within test_gpu_eval_pass.py's tolerance, over several chunks with U not a
multiple of N and over one chunk at 16384 envs; the literal getup path at probability 0 (getup reset with a zero counter and a fall
pool of its own, `pulse_distill_pre_physics`, the step with the recovery counter) gives the pass's frames, flags and sums bit for bit;
the pass's first PD targets are the student's mean action and the teacher does not run; graph and eager runs agree bit for bit; the
student's weights, optimiser and running statistics, the driver's compute, graphs, experience and getup tensors are untouched, the reset
into training is the getup reset on the pass's last terminate flags, and training runs on afterwards replaying its graphs; the PMCP
weights follow the oracle's failed keys."""
import dataclasses

import numpy as np
import pytest
import torch

from tests.test_gpu_eval_pass import DEV, TABLE_KEYS, SynthDataset, _eval, _oracle, _physics, _sim

pytestmark = pytest.mark.gpu
P_REC, P_FALL, REC_STEPS = 0.5, 0.3, 5
T = 4
GETUP_TENSORS = ("recovery_counter", "available_fall_states", "fall_id_assignments", "fall_root_states", "fall_dof_pos", "fall_dof_vel")
EXPERIENCE = ("obses", "kin_gt", "mus", "kin_progress", "rewards", "dones")


def _getup(n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    fall_dof = torch.randn(n, 69, 2, device=DEV, generator=g)       # an env holds at most one fall state: the pool cannot run out
    return dict(recovery_counter=torch.zeros(n, dtype=torch.int32, device=DEV), available_fall_states=torch.zeros(n, dtype=torch.long, device=DEV),
                fall_id_assignments=torch.zeros(n, dtype=torch.long, device=DEV), fall_root_states=torch.randn(n, 13, device=DEV, generator=g),
                fall_dof_pos=fall_dof[..., 0], fall_dof_vel=fall_dof[..., 1], recovery_prob=P_REC, fall_prob=P_FALL, recovery_steps=REC_STEPS)


def _driver(n, seed=3, use_graphs=True):
    from pulse_b200.distill import DistillStepsB200
    from pulse_b200.humanoid_im import HumanoidImCompute
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.vae import PulseVAE, TeacherPNN
    tb, sim = _sim(n, seed)
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in TABLE_KEYS + ("lengths", "num_frames", "dt", "length_starts")}, device=DEV)
    g = torch.Generator().manual_seed(seed + 1)
    pd_off, pd_scale = torch.randn(69, generator=g).to(DEV), (0.5 + torch.rand(69, generator=g)).to(DEV)
    freeze = torch.zeros(69, dtype=torch.uint8)
    freeze[[9, 10, 11, 66, 67, 68]] = 1
    vae = PulseVAE(device=DEV, horizon=T, with_critic=False, seed=seed)                     # im_z_fit.yaml widths
    vae.obs_rms.running_mean.copy_(0.1 * torch.randn(vae.obs_size, generator=g, dtype=torch.float64))
    vae.obs_rms.running_var.copy_(0.5 + torch.rand(vae.obs_size, generator=g, dtype=torch.float64))
    vae.obs_rms._refresh()
    teacher = TeacherPNN(device=DEV, prim_units=(1024, 512), composer_units=(1024, 512), num_prim=3, seed=seed + 1)
    d = DistillStepsB200(HumanoidImCompute(ml), vae, teacher, sim, _getup(n, seed + 7), horizon=T, pd_offset=pd_off, pd_scale=pd_scale,
                         pd_freeze=freeze.to(DEV), use_graphs=use_graphs, reset_seed=5)
    d.first_observation()
    return d


# ------------------------------------------------------------------------------------------------ exact tracking
def test_exact_tracking_gives_zero_metrics():
    N, U = 64, 150
    ds = SynthDataset(U, seed=7)
    _, out, _ = _eval(_driver(N), ds, rate=0.0)
    info = out["eval_info"]
    assert out["chunks"] == 3 and ds.loads == 3
    assert info["eval_success_rate"] == 1.0 and len(out["failed_keys"]) == 0 and len(out["success_keys"]) == U
    for k in ("eval_mpjpe_all", "eval_mpjpe_succ", "mpjpel_all", "mpjpel_succ", "vel_dist", "accel_dist"):
        assert info[k] == 0.0, (k, info[k])
    assert abs(info["mpjpe_pa"]) < 1e-3, info["mpjpe_pa"]


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("N,U,rate,max_frames", [(64, 150, 0.02, 120), (16384, 3000, 0.03, 40)])
def test_pass_matches_oracle(N, U, rate, max_frames):
    ds = SynthDataset(U, seed=11, max_frames=max_frames, spread=max_frames - 5)
    _, out, chunks = _eval(_driver(N), ds, rate=rate, record=True)
    info, steps = _oracle(chunks, N, U, ds._motion_data_keys)
    assert out["chunks"] == len(chunks) == -(-U // N)
    assert out["steps"] == steps
    failed = sorted(np.asarray(info["failed_keys"]).tolist())
    assert sorted(out["failed_keys"].tolist()) == failed
    assert sorted(out["success_keys"].tolist()) == sorted(np.asarray(info["success_keys"]).tolist())
    assert 0 < len(failed) < U                                                     # the student's PD targets decide: some fail, some do not
    for k, v in info["eval_info"].items():
        got = out["eval_info"][k]
        assert abs(got - v) <= 2e-4 * max(1.0, abs(v)), (k, got, v)


# ------------------------------------------------------------------------------------------------ the getup path at probability 0
def _getup_composition(ev, d, seed):
    """Replaces the pass's reset / action / step by the literal HumanoidImGetup path at zero probabilities, eagerly: `reset_getup`
    (own zero recovery counter and fall pool) + the observation of the reset envs, the student's mean action into
    `pulse_distill_pre_physics`, the fused step with the recovery counter."""
    from pulse_b200 import _lib
    n, vae = ev.n, d.vae
    g = _getup(n, seed)
    kin_progress = torch.zeros(n, dtype=torch.int64, device=DEV)
    seen = {"ref": 0, "other": 0}

    def reset():
        s = ev.sim
        ws = ev.comp.reset_getup(motion_ids=ev.motion_ids, motion_start_times=ev.motion_start_times, motion_start_offset=ev.motion_start_offset,
                                 global_offset=ev.global_offset, progress_buf=ev.progress_buf, root_states=s["root_states"], dof_pos=s["dof_pos"],
                                 dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=ev.reset_buf, terminate_buf=ev.terminate_buf,
                                 recovery_counter=g["recovery_counter"], available_fall_states=g["available_fall_states"],
                                 fall_id_assignments=g["fall_id_assignments"], fall_root_states=g["fall_root_states"], fall_dof_pos=g["fall_dof_pos"],
                                 fall_dof_vel=g["fall_dof_vel"], recovery_prob=0.0, fall_prob=0.0, recovery_steps=REC_STEPS,
                                 contact_forces=s.get("contact_forces"), actor_ids=s.get("actor_ids"), phase=ev.phase, seed=seed, offset=0)
        cc = ws["class_counts"].cpu()
        seen["ref"] += int(cc[0])
        seen["other"] += int(cc[1]) + int(cc[2])
        ev.comp.step(body_state=s["body_state"], progress_buf=ev.progress_buf, motion_ids=ev.motion_ids, motion_start_times=ev.motion_start_times,
                     motion_start_offset=ev.motion_start_offset, global_offset=ev.global_offset, obs_buf=ev.obs, env_ids=ws["env_list"],
                     env_count=ws["count"], flags=_lib.STEP_OBS)

    def act():
        mus = vae.eval_actor(ev.obs, use_mean=True)["mus"]
        rc = g["recovery_counter"]
        with torch.cuda.device(DEV):
            _lib.check(ev.lib.pulse_distill_pre_physics(mus.data_ptr(), mus.stride(0), d.pd[0].data_ptr(), d.pd[1].data_ptr(), _lib.ptr(d.pd_freeze),
                                                        n, vae.A, ev.pd_tar.data_ptr(), ev.pd_tar.stride(0), ev.progress_buf.data_ptr(),
                                                        kin_progress.data_ptr(), 1, rc.data_ptr(), _lib.current_stream(DEV)), "pulse_distill_pre_physics")

    def post():
        s = ev.sim
        ev.comp.step(flags=_lib.STEP_ALL, advance=True, obs_buf=ev.obs, rew_buf=ev.rew, reset_buf=ev.reset_buf, terminate_buf=ev.terminate_buf,
                     dof_force=s.get("dof_force"), dof_vel=s["dof_vel"], recovery_counter=g["recovery_counter"], **ev._state())
        times = ev.progress_buf * ev.cfg.dt + ev.motion_start_times + ev.motion_start_offset
        ev.body_pos_gt = ev.comp.motion_lib.get_motion_state(ev.motion_ids, times, offset=ev.global_offset)["rg_pos"]
        ev.metrics.step(s["body_state"][:, :, 0:3], ev.body_pos_gt, ev.terminate_buf)
        assert int(g["recovery_counter"].abs().sum()) == 0                          # the counter stays identically 0

    ev._reset, ev._act, ev._post = reset, act, post
    return seen


def test_getup_path_at_probability_zero_is_the_pass():
    N, U = 64, 150
    from pulse_b200.evaluation import EvalStepsB200
    runs = []
    for literal in (False, True):
        d = _driver(N)
        ev = EvalStepsB200(d, use_graphs=not literal)
        ev.physics = _physics(ev, 0.02)
        seen = _getup_composition(ev, d, seed=23) if literal else None
        frames = []
        ev.record = lambda pos, gt, term: frames.append((pos.clone(), gt.clone(), term.clone()))
        out = ev.run(SynthDataset(U, seed=29))
        torch.cuda.synchronize()
        runs.append((out, frames, seen))
    (a, fa, _), (b, fb, seen) = runs
    assert seen["ref"] > N * a["chunks"] and seen["other"] == 0                      # envs reset inside the chunks, all reference-state
    assert a["steps"] == b["steps"] and len(fa) == len(fb) and int(a["terminated"].sum()) > 0
    for i, (x, y) in enumerate(zip(fa, fb)):
        for u, v in zip(x, y):
            assert torch.equal(u, v), i
    assert np.array_equal(a["terminated"], b["terminated"])
    assert np.array_equal(a["per_sequence"]["sums"], b["per_sequence"]["sums"])
    assert np.array_equal(a["per_sequence"]["counts"], b["per_sequence"]["counts"])


# ------------------------------------------------------------------------------------------------ student and teacher
def test_student_mean_action_and_no_teacher():
    from pulse_b200.vae import pd_targets
    N, U = 64, 150
    d = _driver(N)
    d.play_steps()                                                                  # the experience buffers hold a horizon
    torch.cuda.synchronize()
    before = {k: getattr(d, k).clone() for k in EXPERIENCE}
    first = {}

    def no_teacher(*a, **k):
        raise AssertionError("the teacher ran in the student's evaluation pass")

    from pulse_b200.evaluation import EvalStepsB200
    ev = EvalStepsB200(d)
    stand_in = _physics(ev, 0.02)

    def physics(t):                                   # the first step of the pass: the PD targets of the reset observation
        if not first:
            first.update(obs=ev.obs.clone(), pd_tar=ev.pd_tar.clone())
        stand_in(t)
    ev.physics = physics
    d.teacher.gt_action = no_teacher
    try:
        ev.run(SynthDataset(U, seed=31))
    finally:
        del d.teacher.gt_action
    ref = pd_targets(d.vae.eval_actor(first["obs"], use_mean=True)["mus"], d.pd[0], d.pd[1], freeze=d.pd_freeze)
    torch.cuda.synchronize()
    assert torch.equal(first["pd_tar"], ref)
    assert float(ref.abs().max()) > 0
    for k in EXPERIENCE:
        assert torch.equal(before[k], getattr(d, k)), k


# ------------------------------------------------------------------------------------------------ graph against eager
@pytest.mark.parametrize("rate", [None, 0.02])
def test_graph_equals_eager(rate):
    N, U = 64, 150
    runs = []
    for graphs in (True, False):
        _, out, _ = _eval(_driver(N), SynthDataset(U, seed=13), rate=rate, use_graphs=graphs)
        runs.append(out)
    a, b = runs
    assert a["steps"] == b["steps"] and np.array_equal(a["terminated"], b["terminated"])
    assert np.array_equal(a["per_sequence"]["sums"], b["per_sequence"]["sums"])
    assert np.array_equal(a["per_sequence"]["counts"], b["per_sequence"]["counts"])


# ------------------------------------------------------------------------------------------------ isolation and the reset into training
def _snapshot(d):
    vae, f = d.vae, d.vae.flat
    out = {"params": f.params, "exp_avg": f.exp_avg, "exp_avg_sq": f.exp_avg_sq, "step": f.step, "logstd": vae.logstd,
           "obs_mean": vae.obs_rms.running_mean, "obs_var": vae.obs_rms.running_var, "obs_count": vae.obs_rms.count,
           "value_mean": vae.value_rms.running_mean, "value_var": vae.value_rms.running_var, "value_count": vae.value_rms.count,
           "termination_distances": d.comp.termination_distances}
    out.update({k: getattr(d, k) for k in EXPERIENCE})
    out.update({k: d.getup[k] for k in GETUP_TENSORS})
    return {k: v.clone() for k, v in out.items()}


SIM_STATE = ("body_state", "root_all", "dof_state", "progress_buf", "motion_ids", "motion_start_times", "motion_start_offset", "global_offset",
             "cycle_counter")


def test_pass_leaves_training_state_and_resets_into_training(monkeypatch):
    from pulse_b200 import _lib
    from pulse_b200.evaluation import EvalStepsB200
    N, U = 64, 150
    d = _driver(N)

    def iteration():
        d.play_steps(check=True)
        d.train_epoch(0, mini_epochs=1, minibatch=N * T)            # no annealing: the update graph is captured once
    for _ in range(2):                                      # eager, then captured: the driver's graphs exist before the pass
        iteration()
    torch.cuda.synchronize()
    comp, lib, cfg, graphs = d.comp, d.comp.motion_lib, dataclasses.replace(d.comp.cfg), dict(d._graphs)
    before, kld = _snapshot(d), d.vae.kld_coefficient
    at_reset, env_class = [], []
    reset_training = EvalStepsB200._reset_training

    def spy(ev):                                             # the state a pass hands to the reset into training, and the reset's result
        torch.cuda.synchronize()
        at_reset.append((_snapshot(d), {k: ev.sim[k].clone() for k in SIM_STATE}, ev.terminate_buf.clone(), d.vae.rng_offset.clone()))
        reset_training(ev)
        torch.cuda.synchronize()
        at_reset[-1] += (_snapshot(d),)
        env_class.append(d.reset_ws["env_class"].clone())
    monkeypatch.setattr(EvalStepsB200, "_reset_training", spy)
    ds = SynthDataset(U, seed=17)
    d.evaluate(ds, auto_pmcp_soft=True)                                      # one K-step graph per poll
    d.evaluate(ds, physics=lambda t: _physics(d.eval_steps, 0.3)(t), auto_pmcp_soft=True)   # graph segments; many envs terminate
    torch.cuda.synchronize()
    assert len(at_reset) == 2
    for k in before:                                                          # the first pass changed nothing of the driver's
        assert torch.equal(before[k], at_reset[0][0][k]), k
    for k in before:                                                          # the second pass changed nothing either: its getup tensors
        want = at_reset[0][4][k] if k in GETUP_TENSORS else before[k]        # are those the first reset into training left
        assert torch.equal(want, at_reset[1][0][k]), k
    after = _snapshot(d)
    for k in before:
        if k not in GETUP_TENSORS:
            assert torch.equal(before[k], after[k]), k
    assert d.vae.kld_coefficient == kld
    assert d.comp is comp and d.comp.motion_lib is lib and d.comp.cfg == cfg and not d.comp.cfg.use_mean_reset
    assert d._graphs == graphs                                                # same keys, same graph objects

    # the second reset into training against an eager getup reset from the same state, seed, offset and flags
    snap, st, term, off, _ = at_reset[1]
    assert int(term.sum()) > 0
    s = {k: v.clone() for k, v in st.items()}
    s.update(root_states=s["root_all"][:, 0], dof_pos=s["dof_state"][:, :69, 0], dof_vel=s["dof_state"][:, :69, 1])
    g = {k: snap[k].clone() for k in GETUP_TENSORS}
    g.update(recovery_prob=P_REC, fall_prob=P_FALL, recovery_steps=REC_STEPS)
    reset_buf, term_ref, obs = torch.ones(N, dtype=torch.long, device=DEV), term.clone(), torch.zeros_like(d.obs_carry)
    ws = d.comp.reset_getup(motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                            global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
                            dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=reset_buf, terminate_buf=term_ref,
                            recovery_counter=g["recovery_counter"], available_fall_states=g["available_fall_states"],
                            fall_id_assignments=g["fall_id_assignments"], fall_root_states=g["fall_root_states"], fall_dof_pos=g["fall_dof_pos"],
                            fall_dof_vel=g["fall_dof_vel"], recovery_prob=P_REC, fall_prob=P_FALL, recovery_steps=REC_STEPS,
                            cycle_counter=s["cycle_counter"], contact_forces=d.sim.get("contact_forces"), actor_ids=d.sim.get("actor_ids"),
                            seed=d.reset_seed, offset=0, offset_dev=off)
    d.comp.step(body_state=s["body_state"], progress_buf=s["progress_buf"], motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"],
                motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"], obs_buf=obs, env_ids=ws["env_list"],
                env_count=ws["count"], flags=_lib.STEP_OBS)
    torch.cuda.synchronize()
    assert torch.equal(env_class[1], ws["env_class"])
    env_class = env_class[1]
    for k in SIM_STATE:
        assert torch.equal(d.sim[k], s[k]), k
    for k in GETUP_TENSORS:
        assert torch.equal(d.getup[k], g[k]), k
    assert torch.equal(d.obs_carry, obs) and torch.equal(d.reset_buf, reset_buf) and torch.equal(d.terminate_buf, term_ref)
    assert int(d.vae.rng_offset) == int(off) + 1
    rec = env_class == _lib.GETUP_RECOVERY
    assert int(rec.sum()) > 0 and bool((term[rec] == 1).all())               # recovery episodes only on the envs the pass terminated
    assert bool((env_class != 0).all())                                       # every env was reset

    for _ in range(2):
        iteration()
    torch.cuda.synchronize()
    assert d._graphs.keys() == graphs.keys() and all(d._graphs[k] is graphs[k] for k in graphs)   # replayed, not captured again
    assert bool(torch.isfinite(d.obses).all()) and bool(torch.isfinite(d.kin_gt).all())


# ------------------------------------------------------------------------------------------------ PMCP
@pytest.mark.parametrize("soft", [True, False])
def test_pmcp_weights_follow_oracle_failed_keys(soft):
    from pulse_b200.motion_dataset import MotionDatasetB200
    N, U = 64, 150
    ds = SynthDataset(U, seed=19)
    ds.ds._termination_history[::9] = 2.0                   # an earlier pass's failure counts
    hist0 = ds.ds._termination_history.clone()
    _, out, chunks = _eval(_driver(N), ds, rate=0.02, record=True, pmcp={"auto_pmcp": not soft, "auto_pmcp_soft": soft})
    info, _ = _oracle(chunks, N, U, ds._motion_data_keys)
    ref = MotionDatasetB200({k: {} for k in ds._motion_data_keys}, list(range(-1, 23)), np.zeros((24, 3)), device=DEV)
    ref._termination_history = hist0.clone()
    if soft:
        ref.update_soft_sampling_weight(list(info["failed_keys"]))
    else:
        ref.update_hard_sampling_weight(list(info["failed_keys"]))
    assert len(info["failed_keys"]) > 0
    assert torch.equal(ds._sampling_prob, ref._sampling_prob)
    assert torch.equal(ds._termination_history, ref._termination_history) and torch.equal(out["termination_history"], ref._termination_history)
