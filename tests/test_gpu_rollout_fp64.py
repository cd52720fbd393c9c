"""The rollout side of an iteration, element by element, against float64 references fed the kernels' own operands (tests/fp64_ref.py).

What turns observations into the experience buffer the update trains on: the imitation policy's act_into (normalised input, every actor
and critic layer, the head written into a strided experience slice, the sampled actions with injected and with Philox noise, neglogp,
the de-normalised values, the PD targets) and critic_values_into; the distillation teacher's gt_action (primitives, composer and
pnn_compose) and the student's act_into (encoder, the Philox reparameterisation, the decoder into the mus slice), eval_actor(use_mean)
and pulse_distill_pre_physics; GAE, the normalised advantages and the return targets of finish_returns.  Each GEMM link runs in every
GEMM mode -- default, PULSE_GEMM_BN=128, PULSE_GEMM_STAGES=4 -- at M = 16384 and at a ragged M.  A dropped k-block, a bias column
left out, a wrong Philox block, a missing clamp or a discount applied on the wrong step fails here.  Run with -s to print every margin.
"""
import pytest
import torch

from tests.fp64_links import _check_normalized, _check_pads, _merge64, _merge64_tol, _snapshot, check_mlp_eval, check_rms
from tests.fp64_ref import (U32, Report, adv_normalize_ref, check, check_exact, f64, gae_ref, latent_post_ref, pd_targets_exact,
                            philox_pair_normals, pnn_compose_ref, policy_post_ref, reparam_ref, value_unnorm_ref)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
MODES = {"default": {}, "bn128": {"PULSE_GEMM_BN": "128"}, "stages4": {"PULSE_GEMM_STAGES": "4"}}
SIZES = [16384, 2051]
T_SLICES = 4


def _set_mode(monkeypatch, mode):
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)


def _untouched(rep, link, buf, before, t):
    """Every experience slice but t (dim 1 of an env-major buffer) still holds what it held before the call."""
    keep = [i for i in range(buf.shape[1]) if i != t]
    check_exact(rep, f"{link}: slices other than t = {t} untouched", buf[:, keep], before[:, keep])


# ---------------------------------------------------------------------------------------------------------------- imitation policy
def _imitation_policy(seed):
    from pulse_b200.ppo import PPOPolicy
    pol = PPOPolicy(device=DEV, seed=seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 7)
    pol.obs_rms.update(torch.randn(4096, 934, device=DEV, generator=g) * 1.3 + 0.1)      # non-trivial normalisers
    head = pol.critic.layers[-1]
    probe = torch.randn(2048, 934, device=DEV, generator=g) * 1.5 + 0.2
    v = pol.critic_values(probe)       # value_rms is still the identity here
    with torch.no_grad():              # spread the normalised values over [-15, 15]: rows past both clamp bounds, rows inside
        s = 15.0 / float((v - v.median()).abs().max())
        head.weight[0, :head.K] *= s
        head.weight[0, head.K] = head.weight[0, head.K] * s - s * float(v.median())
        head.refresh()
    pol.value_rms.running_mean.fill_(0.7)
    pol.value_rms.running_var.fill_(2.3)
    pol.advance_rng(1000)              # a non-zero device-side Philox offset
    return pol, g


def _check_policy_post(rep, pol, tag, mu, actions, nlp, values, pd_out, pd, value, eps=None, offset=None):
    A = pol.A
    sg = torch.exp(f64(pol.logstd))
    if eps is None:
        n, nt = philox_pair_normals(pol.rng_seed, mu.shape[0], A, offset)
        n, nt = n.to(DEV), nt.to(DEV)
        plain = policy_post_ref(mu, n, pol.logstd)
        rec = (f64(actions) - f64(mu)) / sg
        check(rep, f"{tag} philox draws (a - mu) / sigma", rec, n, nt + plain["actions"][1] / sg)
        ref = policy_post_ref(mu, n, pol.logstd, eps_tol=nt, value=value, value_mean=pol.value_rms.running_mean,
                              value_var=pol.value_rms.running_var, value_eps=pol.value_rms.eps)
    else:
        ref = policy_post_ref(mu, eps, pol.logstd, value=value, value_mean=pol.value_rms.running_mean,
                              value_var=pol.value_rms.running_var, value_eps=pol.value_rms.eps)
    check(rep, f"{tag} actions", actions, *ref["actions"])
    check(rep, f"{tag} neglogp", nlp, *ref["neglogp"])
    check(rep, f"{tag} values (value_unnorm)", values.reshape(-1), ref["values"][0].reshape(-1), ref["values"][1].reshape(-1))
    check_exact(rep, f"{tag} PD targets", pd_out, pd_targets_exact(actions, *pd))


@pytest.mark.parametrize("M", SIZES)
@pytest.mark.parametrize("mode", list(MODES))
def test_imitation_act_into_links_fp64(monkeypatch, mode, M):
    """act_into at t = 0..3 of [M, T, .] experience buffers (slice bases at 0, 4, 8, 12 bytes mod 16 for A = 69): injected eps and
    Philox noise (A = 69: the pairs 32-34 take the kernel's second loop trip), with and without the side stream; then
    critic_values_into(slot=1) with terminate."""
    _set_mode(monkeypatch, mode)
    pol, g = _imitation_policy(seed=M + len(mode))
    A, T = pol.A, T_SLICES
    rep = Report(f"imitation act_into, M={M}, mode={mode}")
    side = torch.cuda.Stream(DEV)
    actions = torch.full((M, T, A), 7.0, device=DEV)
    mus = torch.full((M, T, A), 7.0, device=DEV)
    nlp = torch.full((M, T), 7.0, device=DEV)
    values = torch.full((M, T, 1), 7.0, device=DEV)
    pd_out = torch.full((M, T, A), 7.0, device=DEV)
    pd = (torch.randn(A, device=DEV, generator=g), torch.rand(A, device=DEV, generator=g) * 3)
    snap = _snapshot(pol.flat)
    m32, r32 = pol.obs_rms.mean_f32.clone(), pol.obs_rms.rstd_f32.clone()
    b = pol._buf(M, False)
    try:
        for t, (noise, use_side, step) in enumerate((("eps", False, 0), ("philox", True, 1), ("eps", True, 0), ("philox", False, 3))):
            obs = torch.randn(M, 934, device=DEV, generator=g) * 1.5 + 0.2
            eps = torch.randn(M, A, device=DEV, generator=g) if noise == "eps" else None
            before = [x.clone() for x in (actions, mus, nlp, values, pd_out)]
            pol.act_into(obs, actions=actions[:, t], neglogp=nlp[:, t], mus=mus[:, t], values=values[:, t], pd=(pd[0], pd[1], pd_out[:, t]),
                         eps=eps, rng_step=step, side=side if use_side else None)
            torch.cuda.synchronize()
            tag = f"t={t} {noise}{' side' if use_side else ''}"
            _check_normalized(rep, f"{tag} normalised obs (bf16)", b["x"], obs, m32, r32, pol.obs_size, pol.obs_size)
            check_mlp_eval(rep, f"{tag} actor", pol.actor, snap, b["x"], M, top_out=mus[:, t])
            check_mlp_eval(rep, f"{tag} critic", pol.critic, snap, b["x"], M)
            value = pol.critic._ws[(M, False)]["out"]
            _check_policy_post(rep, pol, tag, mus[:, t], actions[:, t], nlp[:, t], values[:, t], pd_out[:, t], pd, value, eps=eps,
                               offset=int(pol.rng_offset.item()) + step)
            for name, buf, old in zip(("actions", "mus", "neglogp", "values", "pd targets"), (actions, mus, nlp, values, pd_out), before):
                _untouched(rep, f"{tag} {name}", buf, old, t)
        hi, lo = float((f64(value) > 5).double().mean()), float((f64(value) < -5).double().mean())
        assert hi > 0.01 and lo > 0.01 and hi + lo < 0.9, f"clamped above {hi:.3f}, below {lo:.3f}: the clamp is not exercised on both sides"
        # ---- next values: critic_values_into on the second operand / workspace slot, with terminate
        obs = torch.randn(M, 934, device=DEV, generator=g) * 1.5 + 0.2
        term = (torch.rand(M, device=DEV, generator=g) < 0.3).long()
        nxt = torch.full((T, M, 1), 7.0, device=DEV)
        before = nxt.clone()
        pol.critic_values_into(obs, nxt[2].view(-1), terminate=term, slot=1)
        torch.cuda.synchronize()
        x1 = b["x_next"]
        _check_normalized(rep, "next normalised obs (bf16)", x1, obs, m32, r32, pol.obs_size, pol.obs_size)
        check_mlp_eval(rep, "next critic (slot 1)", pol.critic, snap, x1, M, slot=1)
        v1 = pol.critic._ws[(M, False, 1)]["out"]
        ref, tol = value_unnorm_ref(v1, pol.value_rms.running_mean, pol.value_rms.running_var, pol.value_rms.eps, terminate=term[:, None])
        check(rep, "next values (value_post, terminate)", nxt[2], ref, tol)
        check_exact(rep, "next values: other steps untouched", nxt[[0, 1, 3]], before[[0, 1, 3]])
    finally:
        print("\n" + rep.text())


# ------------------------------------------------------------------------------------------------------------------- latent-task policy
@pytest.mark.parametrize("M", SIZES)
@pytest.mark.parametrize("mode", list(MODES))
def test_latent_task_links_fp64(monkeypatch, mode, M):
    """The step of the reach / speed / strike / VR rollouts (LatentStepsB200._act): the policy's heads_into an [M, T, 32] mus slice, the
    frozen prior's z_prior operands and MLP, pulse_latent_post with Philox noise and with the zero noise of the evaluation pass, the decoder,
    and the PD targets of pulse_pd_targets and pulse_ztask_pre_physics.

    Which epilogue the A = 32 head takes (gemm_wgmma.cu, epilogue_maps / launch_gemm): an fp32 head with no bias, activation or other
    output, N = 32 and a row stride of T * 32 floats from a 128 t-byte base, is the plain-fp32 case -- in the default and bn128 modes the
    6-stage ring with its register epilogue and the TMA fp32 store into the strided slice; with PULSE_GEMM_STAGES=4 the launch clears that
    path and the staged epilogue writes the slice.  N = 32 is below the wide tile in every mode: the launch reports a 128-wide tile."""
    from pulse_b200 import _lib
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.vae import PulseVAE, pd_targets
    import ctypes as C
    _set_mode(monkeypatch, mode)
    W, E, T = 361, 32, T_SLICES
    pol = PPOPolicy(obs_size=W, num_actions=E, units=(2048, 1024, 512), act="silu", device=DEV, seed=M + 3)
    vae = PulseVAE(device=DEV, with_critic=False, seed=1)
    g = torch.Generator(device=DEV).manual_seed(M + 17)
    pol.obs_rms.update(torch.randn(4096, W, device=DEV, generator=g) * 1.3 + 0.1)
    vae.obs_rms.update(torch.randn(4096, vae.obs_size, device=DEV, generator=g) * 1.2 + 0.1)
    pol.value_rms.running_mean.fill_(-0.4)
    pol.value_rms.running_var.fill_(0.6)
    pol.advance_rng(77)
    A, S = vae.A, vae.S
    rep = Report(f"latent-task policy, M={M}, mode={mode}")
    snap_p, snap_v = _snapshot(pol.flat), _snapshot(vae.flat)
    pm32, pr32 = pol.obs_rms.mean_f32.clone(), pol.obs_rms.rstd_f32.clone()
    vm32, vr32 = vae.obs_rms.mean_f32.clone(), vae.obs_rms.rstd_f32.clone()
    mus = torch.full((M, T, E), 7.0, device=DEV)
    actions = torch.full((M, T, E), 7.0, device=DEV)
    nlp = torch.full((M, T), 7.0, device=DEV)
    values = torch.full((T, M, 1), 7.0, device=DEV)
    off, sc = torch.randn(A, device=DEV, generator=g), 0.5 + torch.rand(A, device=DEV, generator=g)
    freeze = (torch.arange(A, device=DEV) % 7 == 3).to(torch.uint8)
    b = pol._buf(M, False)
    bv = vae._buf(M)
    lib = _lib.load()
    try:
        for t in range(T):
            obs = torch.randn(M, W, device=DEV, generator=g) * 1.5 + 0.2
            obs[:, 5:9] *= 8.0                                    # self columns past +-5 once normalised: prior_in unclamped, dec_in clamped
            zero_noise = t == 2
            before = [x.clone() for x in (mus, actions, nlp)]
            vals_before = values.clone()
            prior_head, dec_in = vae.z_prior(obs)
            value = pol.heads_into(obs, mus=mus[:, t], side=torch.cuda.Stream(DEV) if t % 2 else None)
            pol.actor.forward(b["x"], out=mus[:, t])              # the head alone once more: the tile width of its launch
            tile = _lib.gemm_last_launch()["tile_n"]
            eps = torch.zeros(M, E, device=DEV) if zero_noise else None
            a = _lib.LatentPostArgs(mu=mus[:, t].data_ptr(), ld_mu=mus.stride(0), logstd=pol.logstd.data_ptr(), seed=pol.rng_seed,
                                    rng_offset=pol.rng_offset.data_ptr(), rng_step=t, latent=E, actions=actions[:, t].data_ptr(),
                                    ld_actions=actions.stride(0), neglogp=nlp[:, t].data_ptr(), ld_neglogp=nlp.stride(0), value=value.data_ptr(),
                                    ld_value=value.stride(0), values_out=values[t].data_ptr(), ld_values=values[t].stride(0),
                                    prior_mu=prior_head.data_ptr(), ld_prior=prior_head.stride(0), z_bf16=dec_in.data_ptr(), ld_z=dec_in.stride(0),
                                    value_mean=pol.value_rms.running_mean.data_ptr(), value_var=pol.value_rms.running_var.data_ptr(),
                                    value_eps=pol.value_rms.eps)
            if eps is not None:
                a.eps, a.ld_eps = eps.data_ptr(), eps.stride(0)
            _lib.check(lib.pulse_latent_post(C.byref(a), M, _lib.current_stream(DEV)), "pulse_latent_post")
            dec = vae.dec.forward(dec_in)
            pd_out = pd_targets(dec, off, sc, freeze=freeze)
            torch.cuda.synchronize()
            tag = f"t={t} {'zero noise' if zero_noise else 'philox'}"
            assert tile == 128, f"the A = 32 head took a {tile}-wide tile"
            _check_normalized(rep, f"{tag} policy normalised obs (bf16)", b["x"], obs, pm32, pr32, W, W)
            check_mlp_eval(rep, f"{tag} actor", pol.actor, snap_p, b["x"], M, top_out=mus[:, t])
            check_mlp_eval(rep, f"{tag} critic", pol.critic, snap_p, b["x"], M)
            # ---- z_prior: the unclamped normalised self observation, the clamped one in the decoder operand, the pads
            _check_normalized(rep, f"{tag} prior_in (unclamped, bf16)", bv["prior_in"], obs[:, :S], vm32[:S], vr32[:S], S, None, clamp=None)
            assert bool((f64(bv["prior_in"][:, :S]).abs() > 5).any()), "no prior_in element past +-5: the missing clamp is not exercised"
            _check_normalized(rep, f"{tag} dec_in self columns (clamped, bf16)", dec_in[:, E:], obs[:, :S], vm32[:S], vr32[:S], S, None)
            check_mlp_eval(rep, f"{tag} prior", vae.prior, snap_v, bv["prior_in"], M)
            # ---- latent_post
            mu = mus[:, t]
            if zero_noise:
                ref = latent_post_ref(mu, eps, pol.logstd, prior_head[:, :E], actions[:, t], value=value, value_mean=pol.value_rms.running_mean,
                                      value_var=pol.value_rms.running_var, value_eps=pol.value_rms.eps)
            else:
                n, nt = philox_pair_normals(pol.rng_seed, M, E, int(pol.rng_offset.item()) + t)
                n, nt = n.to(DEV), nt.to(DEV)
                ref = latent_post_ref(mu, n, pol.logstd, prior_head[:, :E], actions[:, t], eps_tol=nt, value=value,
                                      value_mean=pol.value_rms.running_mean, value_var=pol.value_rms.running_var, value_eps=pol.value_rms.eps)
            check(rep, f"{tag} latent_post actions", actions[:, t], *ref["actions"])
            check(rep, f"{tag} latent_post neglogp", nlp[:, t], *ref["neglogp"])
            check(rep, f"{tag} latent_post values", values[t].reshape(-1), ref["values"][0].reshape(-1), ref["values"][1].reshape(-1))
            check_exact(rep, f"{tag} latent_post z = bf16(prior_mu + a)", dec_in[:, :E], ref["z"])
            for name, buf, old in zip(("mus", "actions", "neglogp"), (mus, actions, nlp), before):
                _untouched(rep, f"{tag} {name}", buf, old, t)
            keep = [i for i in range(T) if i != t]
            check_exact(rep, f"{tag} values: other steps untouched", values[keep], vals_before[keep])
            # ---- decoder and PD targets
            check_mlp_eval(rep, f"{tag} dec", vae.dec, snap_v, dec_in, M)
            check_exact(rep, f"{tag} pd_targets (freeze)", pd_out, pd_targets_exact(dec, off, sc, freeze))
        root = torch.randn(M, 13, device=DEV, generator=g)
        prev = torch.full((M, 3), 7.0, device=DEV)
        pd2 = torch.full((M, A), 7.0, device=DEV)
        p = _lib.ZTaskPrePhysicsArgs(kind=_lib.ZTASK_STRIKE, dofs=A, action=dec.data_ptr(), ld_action=dec.stride(0), pd_offset=off.data_ptr(),
                                     pd_scale=sc.data_ptr(), freeze=freeze.data_ptr(), pd_out=pd2.data_ptr(), ld_pd=pd2.stride(0),
                                     root_states=root.data_ptr(), root_env_stride=root.stride(0), prev_root_pos=prev.data_ptr())
        _lib.check(lib.pulse_ztask_pre_physics(C.byref(p), M, _lib.current_stream(DEV)), "pulse_ztask_pre_physics")
        torch.cuda.synchronize()
        check_exact(rep, "ztask_pre_physics PD targets (freeze)", pd2, pd_targets_exact(dec, off, sc, freeze))
        check_exact(rep, "ztask_pre_physics prev_root_pos", prev, root[:, :3])
        print(f"\nA = 32 head, mode {mode}: {tile}-wide tile")
    finally:
        print("\n" + rep.text())


# ------------------------------------------------------------------------------------------------------------------------ distillation
def _teacher(act, seed=5, **kw):
    from pulse_b200.vae import TeacherPNN
    t = TeacherPNN(device=DEV, seed=seed, composer_act=act, **kw)
    g = torch.Generator(device=DEV).manual_seed(seed)
    t.rms.running_mean.copy_((torch.rand(934, device=DEV, generator=g) - 0.5).double() * 0.4)
    t.rms.running_var.copy_((torch.rand(934, device=DEV, generator=g) + 0.5).double())
    t.rms._refresh()
    return t, g


def _check_teacher(rep, teacher, obs, out, M, tag):
    snap = _snapshot(teacher.flat)
    teacher.gt_action(obs, out=out)
    torch.cuda.synchronize()
    b = teacher._bufs[M]
    _check_normalized(rep, f"{tag} teacher normalised obs (bf16)", b["x"], obs, teacher.rms.mean_f32, teacher.rms.rstd_f32, teacher.obs_size, None)
    for k, col in enumerate(teacher.cols):
        check_mlp_eval(rep, f"{tag} primitive {k}", col, snap, b["x"], M, top_out=b["acts"][k])
    check_mlp_eval(rep, f"{tag} composer", teacher.composer, snap, b["x"], M)
    w = teacher.composer._ws[(M, False)]["out"]
    y, tol = pnn_compose_ref(w, b["acts"], teacher.composer_act)
    check(rep, f"{tag} pnn_compose ({teacher.composer_act})", out, y, tol)


@pytest.mark.parametrize("M", SIZES)
@pytest.mark.parametrize("mode", list(MODES))
def test_distill_links_fp64(monkeypatch, mode, M):
    """The teacher's gt_action at its default widths into a kin_gt slice; the student's act_into (encoder, Philox reparameterisation with
    noise_out, decoder into the mus slice); eval_actor(use_mean=True); pulse_distill_pre_physics with a freeze mask."""
    from pulse_b200 import _lib
    from pulse_b200.vae import PulseVAE
    _set_mode(monkeypatch, mode)
    rep = Report(f"distillation, M={M}, mode={mode}")
    teacher, g = _teacher("silu")
    T, A, t = T_SLICES, teacher.A, 1
    try:
        obs = torch.randn(M, 934, device=DEV, generator=g) * 1.5 + 0.2
        kin_gt = torch.full((M, T, A), 7.0, device=DEV)
        before = kin_gt.clone()
        _check_teacher(rep, teacher, obs, kin_gt[:, t], M, "")
        _untouched(rep, "kin_gt", kin_gt, before, t)
        # ---- student
        vae = PulseVAE(device=DEV, seed=2, with_critic=False)
        E, S = vae.E, vae.S
        vae.obs_rms.update(torch.randn(4096, vae.obs_size, device=DEV, generator=g) * 1.2 + 0.1)
        vae.advance_rng(500)
        snap = _snapshot(vae.flat)
        m32, r32 = vae.obs_rms.mean_f32.clone(), vae.obs_rms.rstd_f32.clone()
        mus = torch.full((M, T, A), 7.0, device=DEV)
        before = mus.clone()
        noise = torch.zeros(M, E, device=DEV)
        step = 2
        vae.act_into(obs, mus=mus[:, t], rng_step=step, noise_out=noise)
        torch.cuda.synchronize()
        b = vae._buf(M)
        _check_normalized(rep, "student normalised obs (bf16)", b["x"], obs, m32, r32, vae.obs_size, None)
        check_exact(rep, "copy_cols prior_in", b["prior_in"][:, :S], b["x"][:, :S])
        check_exact(rep, "copy_cols dec_in self window", b["dec_in"][:, E:E + S], b["x"][:, :S])
        _check_pads(rep, "copy_cols dec_in", b["dec_in"], E + S)
        check_mlp_eval(rep, "enc", vae.enc, snap, b["x"], M)
        head = vae.enc._ws[(M, False)]["out"]
        n, nt = philox_pair_normals(vae.rng_seed, M, E, int(vae.rng_offset.item()) + step)
        n, nt = n.to(DEV), nt.to(DEV)
        check(rep, "reparam philox noise_out", noise, n, nt)
        z, zt = reparam_ref(head, n, "sample", E, vae.clamp, vae.clamp_lo, vae.clamp_hi, noise_tol=nt)
        check(rep, "reparam z (clamped logvar, bf16)", b["dec_in"][:, :E], z, zt)
        check_mlp_eval(rep, "dec", vae.dec, snap, b["dec_in"], M, top_out=mus[:, t])
        _untouched(rep, "mus", mus, before, t)
        # ---- eval_actor(use_mean=True): the distillation evaluation's path
        out = vae.eval_actor(obs, use_mean=True)
        torch.cuda.synchronize()
        check_mlp_eval(rep, "eval enc", vae.enc, snap, b["x"], M)
        zm, _ = reparam_ref(out["enc_head"], None, "mean", E)
        check_exact(rep, "use_mean z = bf16(mu)", b["dec_in"][:, :E], zm.to(BF))
        check_mlp_eval(rep, "eval dec", vae.dec, snap, b["dec_in"], M, top_out=out["mus"])
        # ---- pulse_distill_pre_physics: PD targets with frozen dofs, kin_progress, the recovery counter
        off, sc = torch.randn(A, device=DEV, generator=g), torch.rand(A, device=DEV, generator=g) * 3
        freeze = (torch.arange(A, device=DEV) % 5 == 0).to(torch.uint8)
        pd_out = torch.full((M, A), 7.0, device=DEV)
        progress = torch.randint(0, 1000, (M,), device=DEV, generator=g)
        kin_progress = torch.full((M, T), -1, dtype=torch.int64, device=DEV)
        rc = torch.randint(0, 4, (M,), device=DEV, generator=g).to(torch.int32)
        rc0 = rc.clone()
        lib = _lib.load()
        _lib.check(lib.pulse_distill_pre_physics(mus[:, t].data_ptr(), mus.stride(0), off.data_ptr(), sc.data_ptr(), freeze.data_ptr(), M, A,
                                                 pd_out.data_ptr(), pd_out.stride(0), progress.data_ptr(), kin_progress[:, t].data_ptr(),
                                                 kin_progress.stride(0), rc.data_ptr(), _lib.current_stream(DEV)), "pulse_distill_pre_physics")
        torch.cuda.synchronize()
        check_exact(rep, "distill PD targets (freeze)", pd_out, pd_targets_exact(mus[:, t], off, sc, freeze))
        check_exact(rep, "kin_progress[:, t]", kin_progress[:, t], progress)
        check_exact(rep, "kin_progress other slices", kin_progress[:, [0, 2, 3]], torch.full_like(kin_progress[:, [0, 2, 3]], -1))
        check_exact(rep, "recovery counter decrement", rc, torch.clamp(rc0 - 1, min=0))
    finally:
        print("\n" + rep.text())


@pytest.mark.parametrize("act", ["relu", None])
def test_teacher_composer_activations_fp64(act):
    """The ReLU and no-activation composers at one small ragged M."""
    M = 300
    teacher, g = _teacher(act, seed=11)
    rep = Report(f"teacher gt_action, composer {act}, M={M}")
    try:
        obs = torch.randn(M, 934, device=DEV, generator=g) * 1.5 + 0.2
        out = torch.full((M, teacher.A), 7.0, device=DEV)
        _check_teacher(rep, teacher, obs, out, M, f"{act}")
        w = f64(teacher.composer._ws[(M, False)]["out"])
        assert bool((w < 0).any() and (w > 0).any()), "the composer weights do not take both signs"
    finally:
        print("\n" + rep.text())


# ------------------------------------------------------------------------------------------------------------------ GAE and returns
class _ValueNorm:
    """What finish_returns reads of a policy: its value normaliser."""

    def __init__(self):
        from pulse_b200.ppo import RunningMeanStdB200
        self.value_rms = RunningMeanStdB200(1, DEV)
        self.value_rms.running_mean.fill_(1.5)
        self.value_rms.running_var.fill_(40.0)
        self.value_rms.count.fill_(3000.0)
        self.value_rms._refresh()


def _rollout(T, N, g):
    r = torch.randn(T, N, device=DEV, generator=g) * 10
    r[:, ::7] *= 100                                                          # rewards up to about +-1e3
    v = torch.randn(T, N, device=DEV, generator=g) * 3 + 1
    nv = torch.randn(T, N, device=DEV, generator=g) * 3 + 1
    d = (torch.rand(T, N, device=DEV, generator=g) < 0.1).float()
    d[:, 1::11] = 1.0                                                         # done at every step
    d[:, 2::11] = 0.0
    d[0, 2::11] = 1.0                                                         # done only at t = 0
    d[:, 3::11] = 0.0
    d[T - 1, 3::11] = 1.0                                                     # done only at t = T-1
    d[:, 4::11] = 0.0                                                         # never done: the longest discounted chains
    return r, v, nv, d


@pytest.mark.parametrize("T,N", [(1, 5), (17, 1027), (32, 16384), (64, 33)])
def test_gae_and_return_targets_fp64(T, N):
    from pulse_b200.rollout import discount_values, finish_returns
    g = torch.Generator(device=DEV).manual_seed(T * 100003 + N)
    gamma, tau = 0.99, 0.95
    r, v, nv, d = _rollout(T, N, g)
    rep = Report(f"GAE and return targets, T={T}, N={N}")
    env_major = lambda x: x.T.reshape(-1)
    try:
        adv_raw, ret_raw = discount_values(d, v, r, nv, gamma=gamma, tau=tau)
        torch.cuda.synchronize()
        a64, ta, r64, tr = gae_ref(r, v, nv, d, gamma, tau)
        check(rep, "GAE advantages (env-major)", adv_raw, env_major(a64), env_major(ta))
        check(rep, "GAE returns (env-major)", ret_raw, env_major(r64), env_major(tr))
        vn = _ValueNorm()
        rms = vn.value_rms
        start = (f64(rms.running_mean).clone(), f64(rms.running_var).clone(), float(rms.count))
        adv_out, ret_out = torch.full((N * T,), 7.0, device=DEV), torch.full((N * T,), 7.0, device=DEV)
        for call in range(2):            # the second call on the same buffers: the advantage statistics start from zero again
            if call == 1:
                start = (f64(rms.running_mean).clone(), f64(rms.running_var).clone(), float(rms.count))
            finish_returns(vn, d.unsqueeze(-1), v.unsqueeze(-1), r.unsqueeze(-1), nv.unsqueeze(-1), adv_out, ret_out, gamma, tau)
            torch.cuda.synchronize()
            y, tol = adv_normalize_ref(adv_raw)
            check(rep, f"call {call} normalised advantages", adv_out, y, tol)
            # returns: normalised with the statistics that include the values batch, clamped to +-5; then merged themselves
            vals = v.reshape(-1, 1)
            mean, var, _, _, _ = _merge64(*start, vals)
            em, ev = _merge64_tol(*start, vals)
            m32, sd = float(mean.float()), float(torch.sqrt(var.float() + rms.eps))
            x = f64(ret_raw)
            yu = (x - m32) / sd
            yr = torch.clamp(yu, -5.0, 5.0)
            # fp32(mean) and fp32(sqrt(fp32(var) + eps)) may each round the other way; then the difference and the quotient.  The clamp
            # is 1-Lipschitz, so the bound of the unclamped quotient holds for the clamped one.
            e_m = float(em) + 2 * U32 * abs(m32)
            e_sd = 0.5 * (float(ev) + 2 * U32 * float(var)) / sd + 2 * U32 * sd
            tol_r = (U32 * (x - m32).abs() + e_m) / sd + yu.abs() * (e_sd / sd + U32)
            inside = yu.abs() < 5.0
            check(rep, f"call {call} normalised returns", ret_out, yr, tol_r)
            check_rms(rep, f"call {call} value_rms", rms, start, [vals, ret_raw.reshape(-1, 1)])
        assert bool((~inside).any()) or T == 1, "no return reaches the +-5 clamp"
    finally:
        print("\n" + rep.text())
