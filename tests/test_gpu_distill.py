"""The distillation rollout on the GPU: `pulse_vae_reparam_philox`, `pulse_distill_pre_physics` and `DistillStepsB200` (one horizon of
HumanoidImDistillGetup with getup resets, the frozen teacher and the VAE student, and the only_kin_loss update).

The driver is checked bit for bit against an eager composition of already-validated calls: `reset_getup` + the observation launch,
`TeacherPNN.gt_action`, `PulseVAE.eval_actor` with the kernel's draws injected, `pd_targets`, a torch recovery decrement and the fused
step kernel."""
import math

import numpy as np
import pytest
import torch

from tests.test_gpu_rollout import DEV, _sim

pytestmark = pytest.mark.gpu
P_REC, P_FALL, REC_STEPS = 0.3, 0.3, 5


def _nets(T, seed=4):
    from pulse_b200.vae import PulseVAE, TeacherPNN
    vae = PulseVAE(device=DEV, horizon=T, with_critic=False, seed=seed)                     # im_z_fit.yaml widths
    teacher = TeacherPNN(device=DEV, prim_units=(1024, 512), composer_units=(1024, 512), num_prim=3, seed=seed + 1)   # env_im_vae.yaml
    return vae, teacher


def _world(n, T, seed=2, graphs=True):
    """Simulator, getup tables and a driver; early termination forced high (tight distance, short episodes) so that reference-state,
    fall and recovery resets all happen inside a horizon."""
    from pulse_b200.distill import DistillStepsB200
    tb, comp, sim = _sim(n, clips=64, seed=seed)
    comp.termination_distances.fill_(0.15)
    comp.cfg.max_episode_length = 24
    g = torch.Generator(device=DEV).manual_seed(seed + 7)
    P = n                              # an env holds at most one fall state: the pool cannot run out
    fall_dof = torch.randn(P, 69, 2, device=DEV, generator=g)
    getup = dict(recovery_counter=torch.zeros(n, dtype=torch.int32, device=DEV), available_fall_states=torch.zeros(P, dtype=torch.long, device=DEV),
                 fall_id_assignments=torch.zeros(n, dtype=torch.long, device=DEV), fall_root_states=torch.randn(P, 13, device=DEV, generator=g),
                 fall_dof_pos=fall_dof[..., 0], fall_dof_vel=fall_dof[..., 1], recovery_prob=P_REC, fall_prob=P_FALL, recovery_steps=REC_STEPS)
    vae, teacher = _nets(T)
    freeze = torch.zeros(69, dtype=torch.uint8, device=DEV)
    freeze[[5, 6, 40]] = 1
    drv = DistillStepsB200(comp, vae, teacher, sim, getup, horizon=T, pd_offset=0.1 * torch.randn(69, device=DEV, generator=g),
                           pd_scale=1.0 + torch.rand(69, device=DEV, generator=g), pd_freeze=freeze, use_graphs=graphs, reset_seed=11)
    drv.first_observation()
    return drv


def _eager_horizon(d, refresh=None, physics=None):
    """One horizon of DistillStepsB200's step, call by call, into d's buffers (d's own play_steps is never called).  Returns the reset-class counts."""
    from pulse_b200 import _lib
    from pulse_b200.vae import pd_targets
    s, g, vae, T, n = d.sim, d.getup, d.vae, d.T, d.n
    counts = torch.zeros(3, dtype=torch.long)
    eps = torch.zeros(n, vae.E, device=DEV)
    scratch = torch.zeros(n, vae.A, device=DEV)
    d.obses[:, 0].copy_(d.obs_carry)
    for t in range(T):
        ws = d.comp.reset_getup(motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                                global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
                                dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=d.reset_buf, terminate_buf=d.terminate_buf,
                                recovery_counter=g["recovery_counter"], available_fall_states=g["available_fall_states"],
                                fall_id_assignments=g["fall_id_assignments"], fall_root_states=g["fall_root_states"], fall_dof_pos=g["fall_dof_pos"],
                                fall_dof_vel=g["fall_dof_vel"], recovery_prob=g["recovery_prob"], fall_prob=g["fall_prob"],
                                recovery_steps=g["recovery_steps"], cycle_counter=s.get("cycle_counter"), contact_forces=s.get("contact_forces"),
                                actor_ids=s.get("actor_ids"), seed=d.reset_seed, offset=t, offset_dev=vae.rng_offset)
        counts += ws["class_counts"].cpu().long()
        if refresh is not None:
            refresh(d, t)
        d.comp.step(body_state=s["body_state"], progress_buf=s["progress_buf"], motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"],
                    motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"], obs_buf=d.obses[:, t], env_ids=ws["env_list"],
                    env_count=ws["count"], flags=_lib.STEP_OBS)
        d.kin_gt[:, t].copy_(d.teacher.gt_action(d.obses[:, t]))
        vae.act_into(d.obses[:, t], mus=scratch, rng_step=t, noise_out=eps)          # only to record the kernel's draws
        d.mus[:, t].copy_(vae.eval_actor(d.obses[:, t], noise=eps)["mus"])
        pd_targets(d.mus[:, t], d.pd[0], d.pd[1], out=d.pd_tar, freeze=d.pd_freeze)
        d.kin_progress[:, t].copy_(s["progress_buf"])
        g["recovery_counter"].copy_(torch.clamp_min(g["recovery_counter"] - 1, 0))
        if physics is not None:
            physics(d, t)
        nxt = d.obses[:, t + 1] if t + 1 < T else d.obs_carry
        d.comp.step(obs_buf=nxt, rew_buf=d.rewards[t], fdones_out=d.dones[t], advance=True, recovery_counter=g["recovery_counter"], **d._step_kw())
    vae.advance_rng(T)
    return counts


EXPERIENCE = ("obses", "obs_carry", "kin_gt", "kin_progress", "mus", "pd_tar", "rewards", "dones", "reset_buf", "terminate_buf")


def _assert_same(a, b, where):
    torch.cuda.synchronize()
    for name in EXPERIENCE:
        assert torch.equal(getattr(a, name), getattr(b, name)), (where, name)
    assert torch.equal(a.sim["progress_buf"], b.sim["progress_buf"]), where
    assert torch.equal(a.sim["body_state"], b.sim["body_state"]), where
    for k in ("recovery_counter", "fall_id_assignments", "available_fall_states"):
        assert torch.equal(a.getup[k], b.getup[k]), (where, k)


# ---------------------------------------------------------------------------------------------------------------------------------------------
def test_reparam_philox_matches_injected_noise_and_is_gaussian():
    vae, _ = _nets(32)
    M, E = 8192, vae.E
    g = torch.Generator(device=DEV).manual_seed(3)
    obs = torch.randn(M, vae.obs_size, device=DEV, generator=g)
    vae.enc.layers[-1].bias[E:] = torch.linspace(-7.0, 4.0, E, device=DEV)   # log-variances on both sides of the clamp [-5, 2]
    mus, eps = torch.zeros(M, 3, vae.A, device=DEV), torch.zeros(M, E, device=DEV)
    vae.act_into(obs, mus=mus[:, 1], rng_step=3, noise_out=eps)
    dec_a = vae._buf(M)["dec_in"].clone()
    ref = vae.eval_actor(obs, noise=eps)                                  # pulse_vae_reparam(Z_SAMPLE) with the same draws
    torch.cuda.synchronize()
    assert torch.equal(dec_a, vae._buf(M)["dec_in"])
    assert torch.equal(mus[:, 1], ref["mus"])
    assert float(mus[:, [0, 2]].abs().max()) == 0.0
    e = eps.double()
    assert abs(float(e.mean())) < 0.01 and abs(float(e.var()) - 1.0) < 0.02
    assert abs(float((e ** 4).mean()) - 3.0) < 0.15
    c = torch.corrcoef(e.t())
    assert float((c - torch.eye(E, device=DEV, dtype=c.dtype)).abs().max()) < 0.06
    draws = []
    for step, bump in ((3, 0), (4, 0), (3, 32)):
        if bump:
            vae.advance_rng(bump)
        out = torch.zeros(M, E, device=DEV)
        vae.act_into(obs, mus=mus[:, 0], rng_step=step, noise_out=out)
        draws.append(out)
    torch.cuda.synchronize()
    assert torch.equal(draws[0], eps)                                     # same (seed, offset, step)
    assert not torch.equal(draws[1], eps) and not torch.equal(draws[2], eps)


def test_pre_physics_kernel():
    from pulse_b200 import _lib
    from pulse_b200.vae import pd_targets
    n, T, t, A = 1000, 5, 2, 69
    g = torch.Generator(device=DEV).manual_seed(8)
    mus = torch.randn(n, T, A, device=DEV, generator=g)
    off, sc = torch.randn(A, device=DEV, generator=g), torch.rand(A, device=DEV, generator=g) * 3
    freeze = (torch.rand(A, device=DEV, generator=g) < 0.2).to(torch.uint8)
    pd = torch.full((n, T, A), -9.0, device=DEV)
    kin = torch.full((n, T), -7, dtype=torch.long, device=DEV)
    prog = torch.randint(0, 300, (n,), device=DEV, generator=g)
    rc0 = torch.randint(0, REC_STEPS + 1, (n,), dtype=torch.int32, device=DEV, generator=g)
    rc0[:3] = torch.tensor([0, 1, REC_STEPS], dtype=torch.int32)
    rc = rc0.clone()
    lib = _lib.load()
    for fr in (None, freeze):
        rc.copy_(rc0)
        with torch.cuda.device(DEV):
            _lib.check(lib.pulse_distill_pre_physics(mus[:, t].data_ptr(), mus.stride(0), off.data_ptr(), sc.data_ptr(), _lib.ptr(fr), n, A,
                                                     pd[:, t].data_ptr(), pd.stride(0), prog.data_ptr(), kin[:, t].data_ptr(), kin.stride(0),
                                                     rc.data_ptr(), _lib.current_stream(DEV)), "pulse_distill_pre_physics")
        ref = pd_targets(mus[:, t], off, sc, freeze=fr)
        torch.cuda.synchronize()
        assert torch.equal(pd[:, t], ref)
        assert torch.equal(kin[:, t], prog)
        assert torch.equal(rc, torch.clamp_min(rc0 - 1, 0)) and rc[:3].tolist() == [0, 0, REC_STEPS - 1]
        keep = [i for i in range(T) if i != t]
        assert bool((pd[:, keep] == -9.0).all()) and bool((kin[:, keep] == -7).all())


@pytest.mark.parametrize("n", [2051, 8192])
def test_horizon_matches_eager_composition(n):
    """Single-graph driver (teacher on the side stream) vs the eager composition over four horizons: eager first use, capture, replays.
    A second driver with the same seeds produces the same experience."""
    T = 32
    drv, twin, ref = _world(n, T), _world(n, T), _world(n, T, graphs=False)
    counts = torch.zeros(3, dtype=torch.long)
    for it in range(4):
        drv.play_steps(check=True)
        twin.play_steps()
        counts += _eager_horizon(ref)
        _assert_same(drv, ref, ("horizon", it))
        _assert_same(drv, twin, ("twin", it))
    assert bool((counts > 0).all()), counts.tolist()                       # reference-state, fall and recovery resets all occurred
    assert ("horizon", True) in drv._graphs and not isinstance(drv._graphs[("horizon", True)], bool)


def test_hooks_segment_mode_matches_eager_composition():
    """With physics(t) / refresh(t, ws) the horizon runs as graph segments between the hook calls; the same callbacks at the same points of
    the eager composition give the same experience."""
    n, T = 1024, 8

    def refresh(d, t, ws=None):        # the simulator's refresh: the rigid-body root follows the (reset) root state
        d.sim["body_state"][:, 0, :7].copy_(d.sim["root_states"][:, :7])

    def physics(d, t):                 # a deterministic stand-in for the simulation step, driven by the PD targets
        d.sim["root_states"][:, :3].add_(0.001 * d.pd_tar[:, :3])
        d.sim["body_state"][:, :24, :3].add_(0.5 * d.sim["root_states"][:, None, :3] * 1e-3)

    drv, ref = _world(n, T), _world(n, T, graphs=False)
    drv.refresh = lambda t, ws: refresh(drv, t, ws)
    drv.physics = lambda t: physics(drv, t)
    for it in range(3):
        drv.play_steps()
        _eager_horizon(ref, refresh=refresh, physics=physics)
        _assert_same(drv, ref, ("segments", it))
    assert not isinstance(drv._graphs[("act", 0, True)], bool)


def _rms_reference(batches, init):
    """RunningMeanStd's training-mode merges (rms_merge_kernel) over `batches` in float64 from exact batch sums (math.fsum of the fp32
    values and of their exact float64 squares), with a bound on the device's deviation: its sums add n fp64 terms in some order
    ((n - 1) u64 of the sum of magnitudes), then every merge operation rounds once; errors carried from merge to merge."""
    u = 2.0 ** -53
    mean, var, cnt = (t.cpu().double().numpy().copy() for t in init)
    cnt = float(cnt)
    e_mean, e_var = np.zeros_like(mean), np.zeros_like(var)
    for x in batches:
        x = x[:, :mean.shape[0]].cpu().double().numpy()
        n = x.shape[0]
        s = np.array([math.fsum(col) for col in x.T])
        q = np.array([math.fsum(col) for col in (x * x).T])
        e_s, e_q = (n - 1) * u * np.abs(x).sum(0) + u * np.abs(s), (n - 1) * u * q + u * q
        tot = cnt + n
        bm = s / n
        e_bm = e_s / n + u * np.abs(bm)
        bv = (q - n * bm * bm) / (n - 1)
        e_bv = (e_q + 2 * n * np.abs(bm) * e_bm + 4 * u * (q + n * bm * bm)) / (n - 1) + u * np.abs(bv)
        delta = bm - mean
        e_d = e_bm + e_mean + u * np.abs(delta)
        m2 = var * cnt + bv * n + delta * delta * cnt * n / tot
        e_m2 = (e_var * cnt + e_bv * n + 2 * np.abs(delta) * e_d * cnt * n / tot
                + 8 * u * (var * cnt + np.abs(bv) * n + delta * delta * cnt * n / tot))
        e_mean = e_mean + e_d * n / tot + 4 * u * (np.abs(mean) + np.abs(delta))
        mean = mean + delta * n / tot
        var = m2 / tot
        e_var = e_m2 / tot + u * np.abs(var)
        cnt = tot
    return mean, var, cnt, e_mean, e_var


def test_train_epoch_matches_eager_optimize_kin_and_ar1_mask():
    """train_epoch (graphs, re-captured when annealing changes the KL coefficient) against the same sequence of eager optimize_kin calls.
    The first minibatch, before any weight update, is bit-identical.  After that `optimize_kin` is not bitwise reproducible even
    eagerly (bias gradients and batch moments are sums accumulated with atomics in scheduling order), so the driver must stay as close
    to one eager run as a second eager run does."""
    n, T, mb, mini = 512, 32, 4096, 3
    drv = _world(n, T)
    for _ in range(2):
        drv.play_steps()
    rows = n * T
    obs, gt, prog = drv.obses.view(rows, -1), drv.kin_gt.view(rows, -1), drv.kin_progress.view(rows)
    runs = [_nets(T)[0] for _ in range(2)]
    init_rms = [t.clone() for t in (runs[0].obs_rms.running_mean, runs[0].obs_rms.running_var, runs[0].obs_rms.count)]
    for t, u in zip(init_rms, (drv.vae.obs_rms.running_mean, drv.vae.obs_rms.running_var, drv.vae.obs_rms.count)):
        assert torch.equal(t, u)                    # the driver's statistics start where a fresh network's do
    stats = {0: [], 1: [], "drv": []}
    ar1 = []
    for epoch in (3000, 3001):                 # past epoch 2500 annealing changes the KL coefficient: graphs are captured anew
        torch.manual_seed(epoch)
        stats["drv"].append(drv.train_epoch(epoch, mini_epochs=mini, minibatch=mb).clone().view(-1, 8))
        for r, vae_e in enumerate(runs):
            torch.manual_seed(epoch)
            for k in range(mini):
                for i in range(rows // mb):
                    s = vae_e.optimize_kin(obs[i * mb:(i + 1) * mb], gt[i * mb:(i + 1) * mb], prog[i * mb:(i + 1) * mb], update_obs_rms=True)
                    stats[r].append(s.clone())
                    if r == 0:
                        head = vae_e.enc._ws[(mb, True)]["out"]
                        ar1.append((head[:, :vae_e.E].clone(), prog[i * mb:(i + 1) * mb].clone(), float(s[2])))
                    vae_e.anneal(epoch)
    torch.cuda.synchronize()
    st_d, st_0, st_1 = torch.cat(stats["drv"]), torch.stack(stats[0]), torch.stack(stats[1])
    assert torch.equal(st_d[0], st_0[0]) and torch.equal(st_1[0], st_0[0])
    a, b, c = drv.vae, runs[0], runs[1]
    assert a.kld_coefficient == b.kld_coefficient < 0.01

    def within_eager_spread(x, y, z, name):
        spread = float((z - y).abs().max())
        if spread == 0.0:
            assert torch.equal(x, y), name
        else:
            assert float((x - y).abs().max()) <= 10.0 * spread, (name, float((x - y).abs().max()), spread)

    within_eager_spread(st_d, st_0, st_1, "stats")
    for name in ("params", "exp_avg", "exp_avg_sq"):
        within_eager_spread(getattr(a.flat, name), getattr(b.flat, name), getattr(c.flat, name), name)
    # The running observation statistics: the batch moments are fp64 atomics in scheduling order, so two runs agree bit for bit only
    # when every column's sum happens to round the same way.  All three are held to the exact float64 merge sequence instead.
    batches = [obs[i * mb:(i + 1) * mb] for _ in range(2 * mini) for i in range(rows // mb)]
    ref_mean, ref_var, ref_count, e_mean, e_var = _rms_reference(batches, init_rms)
    for run in (a, b, c):
        assert float(run.obs_rms.count) == ref_count
        for name, ref, err in (("running_mean", ref_mean, e_mean), ("running_var", ref_var, e_var)):
            got = getattr(run.obs_rms, name).cpu().numpy()
            r = np.abs(got - ref) / err
            assert r.max() < 1.0, (name, float(r.max()), int(r.argmax()))
    # the AR(1) term over the recorded progress (amp_agent.py:792-808), restated in fp32
    held = reset = 0
    for mu, p, got in ar1:
        mu, p = mu.view(-1, T, mu.shape[-1]), p.view(-1, T)
        nxt, cur = p[:, 1:], p[:, :-1]
        keep = (nxt - cur == 1) & ~((nxt <= 2) | (cur <= 2))
        held += int((nxt == cur).sum())
        reset += int((nxt < cur).sum())
        norms = torch.linalg.vector_norm(mu[:, 1:] - 0.99 * mu[:, :-1], dim=-1)
        assert abs(float(norms[keep].double().sum()) - got) <= 1e-4 * max(1.0, abs(got))
    assert held > 0 and reset > 0                   # recovery envs held their progress, envs reset inside the horizon
