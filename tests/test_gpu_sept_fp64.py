"""The terrain task's amp_sept policy (pulse_b200/sept.py), link by link, against float64 references fed the kernels' own operands
(tests/fp64_ref.py, tests/fp64_links.py).

Training: one train_minibatch at the production widths (M = 16384, B = 4096), at a ragged M = 5000 / B = 1000, and at the SEPT_SMALL
widths with M = 2051 / B = 683 (E = 24, S = 22, N0 = 96: the embedding window, the two dpre0 halves and every N narrower than one tile),
in the default, PULSE_GEMM_BN=128 and PULSE_GEMM_STAGES=4 modes.  Links: the split normalise and its untouched self window, the headless
task encoder writing SiLU(.) into P[:, :E], every actor / critic forward and SiLU-gated dgrad (the layer-0 dgrads land in the two halves of
dpre0; the critic's N = 1 head runs through the tensor-core GEMM), pulse_ppo_loss, the fused embedding gradient
dEmb = silu'(pre_top) * ([dPre0_actor | dPre0_critic] . [W_a0[:, :E] ; W_c0[:, :E]]) over K = 2 N0, the task encoder's backward from it,
the discriminator chain, every weight-gradient total, Adam and the observation statistics.  The ragged case runs three minibatches
(clipping off / on / off); the second prefetches the third, which runs from operand slot 1 after two Adam steps and is checked as well.
Eval: act() / critic_values() at M = 2051 and 16384, where the wide SiLU forwards take the 128 x 256 tile.
test_gpu_sept.py's cosine checks against fp32 autograd stay; a missing k-block or a half of dpre0 read from the wrong rows passes those and
fails here.  Run with -s to print the margin of every link.
"""
import pytest
import torch

from tests.fp64_links import (_check_adam, _check_pads, _snapshot, _w, check, check_disc, check_grads, check_mlp, check_mlp_eval,
                              check_ppo_loss, check_rms, check_split, merge_chain64, rms_f32)
from tests.fp64_ref import U32, UBF, Gemm, Report, check_exact, f64, gaussian_sample_ref, silu_gated
from tests.sept_fixture import SEPT_FULL, SEPT_SMALL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

CASES = {"full": (SEPT_FULL, 16384, 4096), "ragged": (SEPT_FULL, 5000, 1000), "small": (SEPT_SMALL, 2051, 683)}
MODES = {"default": {}, "bn128": {"PULSE_GEMM_BN": "128"}, "stages4": {"PULSE_GEMM_STAGES": "4"}}


def _new_policy(d, seed):
    from tests.test_gpu_sept import _policy
    pol, _, _, _ = _policy(d, seed=seed)
    pol.disc.rms.frozen = False
    head = pol.actor.layers[-1]
    with torch.no_grad():             # bias a few action heads past the soft bound so the bounds loss has active elements
        head.weight[:4, head.K] = torch.tensor([1.5, -1.5, 1.2, -1.2], device=DEV)
        head.refresh()
    g = torch.Generator(device=DEV).manual_seed(seed + 100)
    pol.obs_rms.update(torch.randn(4096, pol.obs_size, device=DEV, generator=g) * 1.3 + 0.1)      # non-trivial normalisers
    pol.disc.rms.update(torch.randn(4096, pol.disc.size, device=DEV, generator=g) * 0.9 - 0.1)
    return pol, g


def _ppo_inputs(pol, M, B, g):
    """As test_gpu_update_fp64._ppo_inputs: rows in every clip regime, |mu| > 1 on the biased heads."""
    obs = torch.randn(M, pol.obs_size, device=DEV, generator=g) * 1.5 + 0.2
    eps = torch.randn(M, pol.A, device=DEV, generator=g)
    out = pol.act(obs, eps=eps)
    actions, nlp, mus = out["actions"].clone(), out["neglogpacs"].clone(), out["mus"].clone()
    adv = torch.randn(M, device=DEV, generator=g)
    grp = torch.arange(M, device=DEV) % 4
    nlp = nlp + torch.where(grp == 1, 0.4, torch.where(grp == 2, -0.4, torch.where(grp == 3, 0.4, 0.0)))
    adv = torch.where(grp == 1, adv.abs() + 0.1, torch.where(grp >= 2, -(adv.abs() + 0.1), adv))
    ret = torch.randn(M, device=DEV, generator=g)
    amp = tuple(torch.randn(B, pol.disc.size, device=DEV, generator=g) * s + o for s, o in ((1.0, 0.0), (1.3, 0.2), (0.7, 0.3)))
    return obs, actions, nlp, adv, ret, mus, amp


def _rms_state(rms):
    return f64(rms.running_mean).clone(), f64(rms.running_var).clone(), float(rms.count)


def _check_self_window(rep, pol, obs, mean32, rstd32, P, T):
    """P[:, E:] (and T) after the task forward == a separate pulse_normalize_split of the same rows with the same statistics, bit for bit:
    the task net's top epilogue wrote nothing past column E."""
    from pulse_b200 import _lib
    P2, T2 = torch.full_like(P, 3.0), torch.full_like(T, 3.0)
    _lib.check(_lib.load().pulse_normalize_split(obs.data_ptr(), obs.stride(0), obs.shape[0], obs.shape[1], pol.S, mean32.data_ptr(),
                                                 rstd32.data_ptr(), P2.data_ptr(), P2.stride(0), pol.E, T2.data_ptr(), T2.stride(0), None,
                                                 _lib.current_stream(DEV)), "pulse_normalize_split")
    torch.cuda.synchronize()
    check_exact(rep, "self window P[:, E:] after the task forward", P[:, pol.E:], P2[:, pol.E:])
    check_exact(rep, "task operand T after the task forward", T, T2)


def _check_sept_minibatch(rep, pol, M, B, snap, obs_f32, disc_stats, inputs, slot, slack=0.0):
    obs, actions, old_nlp, adv, ret, mus, amp = inputs
    E, S = pol.E, pol.S
    b = pol._buf(M, True)
    P, T = b["x2"][slot], b["t2"][slot]
    check_split(rep, P, T, obs, *obs_f32, E, S, slack)
    if slack == 0.0:                  # the exact statistics the kernel used are known
        _check_self_window(rep, pol, obs, obs_f32[0], obs_f32[1], P, T)
    # ---- task encoder (headless: SiLU into P[:, :E]; its backward starts from dEmb), actor, critic
    wt, bt = check_mlp(rep, "task", pol.task, snap, T, b["demb"], M, top_out=P[:, :E])
    wa, ba = check_mlp(rep, "actor", pol.actor, snap, P, b["dmu"], M)
    top = len(pol.critic.layers) - 1
    assert not pol.critic._head1(top), "the critic's N = 1 head after a SiLU layer must run through the tensor-core GEMM"
    wc, bc = check_mlp(rep, "critic", pol.critic, snap, P, b["dv"], M)
    n_amb = check_ppo_loss(rep, pol, M, actions, old_nlp, adv, ret, mus)
    # ---- the embedding gradient of both consumers: one dgrad over K = 2 N0, B MN-major from [W_a0 ; W_c0] as they were before the call
    a0, c0 = pol.actor.layers[0], pol.critic.layers[0]
    n0 = a0.N
    w_cat = torch.cat([_w(snap, pol.flat, a0)[:, :E], _w(snap, pol.flat, c0)[:, :E]])
    y, acc = silu_gated(Gemm(b["dpre0"][:M, :2 * n0], w_cat), pol.task.top_preact(M)[:M, :E])
    check(rep, "dEmb = silu'(task top pre) * (dpre0 . [W_a0 ; W_c0][:, :E])", b["demb"][:M, :E], y, acc * (1 + UBF) + UBF * y.abs())
    _check_pads(rep, "dEmb", b["demb"][:M], E)
    check_disc(rep, pol, B, snap, disc_stats, amp, slot)
    check_grads(rep, "task", pol.task, wt, bt)
    check_grads(rep, "actor", pol.actor, wa, ba)
    check_grads(rep, "critic", pol.critic, wc, bc)
    return n_amb


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", list(MODES))
def test_sept_update_links_fp64(monkeypatch, mode, case):
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    d, M, B = CASES[case]
    pol, g = _new_policy(d, seed=M + B)
    rep = Report(f"SeptPolicy update, {case}: M={M}, B={B}, E={pol.E}, S={pol.S}, N0={pol.actor.layers[0].N}, mode={mode}")
    steps = 3 if case == "ragged" else 1
    obs0, disc0 = _rms_state(pol.obs_rms), _rms_state(pol.disc.rms)
    norm1, inputs, note = None, [], ""
    try:
        for step in range(steps):
            while len(inputs) < (1 if step == 0 else steps):     # the third minibatch is made before the second call, which prefetches it
                inputs.append(_ppo_inputs(pol, M, B, g))
            obs, actions, old_nlp, adv, ret, mus, amp = inputs[step]
            snap = _snapshot(pol.flat)
            obs_f32 = (pol.obs_rms.mean_f32.clone(), pol.obs_rms.rstd_f32.clone())
            disc_stats = _rms_state(pol.disc.rms)
            if steps > 1:      # clipping off, on, off: max_norm far above, then far below the norm of the first step's gradients
                pol.grad_norm = 0.25 * norm1 if step == 1 else 1e9
            kw = {}
            if steps > 1 and step == 1:
                kw = dict(prefetch=(inputs[2][0], inputs[2][6]))
            elif steps > 1 and step == 2:
                kw = dict(slot=1, prepared=True)
            pol.reset_stats()
            pol.train_minibatch(obs, actions, old_nlp, adv, ret, old_mu=mus, amp=amp, keep_grads=True, **kw)
            torch.cuda.synchronize()
            if step == 0:
                n_amb = _check_sept_minibatch(rep, pol, M, B, snap, obs_f32, disc_stats, inputs[0], 0)
                check_rms(rep, "obs_rms after minibatch 1", pol.obs_rms, obs0, [obs])
                norm1 = float(f64(pol.flat.grads).norm())
            elif step == 2:
                # operand slot 1 was prepared during the second call with the statistics merged through minibatch 2: their fp32 values
                # from the fp64 merge chain, which may round the last bit the other way from the device's own merges (4 u32 slack)
                f32 = rms_f32(*obs0, [inputs[0][0], inputs[1][0]])
                chain = [x for i in (0, 1) for x in inputs[i][6]]
                mean, _, var, _, cnt = merge_chain64(*disc0, chain)
                n_amb = max(n_amb, _check_sept_minibatch(rep, pol, M, B, snap, f32, (mean, var, cnt), inputs[2], 1, slack=4 * U32))
                check_rms(rep, "obs_rms after minibatch 3", pol.obs_rms, obs0, [x[0] for x in inputs])
                check_rms(rep, "disc rms after minibatch 3", pol.disc.rms, disc0, [x for i in range(3) for x in inputs[i][6]])
            _check_adam(rep, pol.flat, snap, pol.grad_norm, pol.lr, f"step {step + 1}", expect_clip=(step == 1) if steps > 1 else None)
        note = f"\n  PPO rows excluded as ambiguous: {n_amb} of {M} (largest over the checked minibatches)"
    finally:
        print("\n" + rep.text() + note)


@pytest.mark.parametrize("M", [2051, 16384])
@pytest.mark.parametrize("mode", ["default", "bn128"])
def test_sept_eval_links_fp64(monkeypatch, mode, M):
    from pulse_b200 import _lib
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    d = SEPT_FULL
    pol, g = _new_policy(d, seed=M)
    E = pol.E
    obs = torch.randn(M, pol.obs_size, device=DEV, generator=g) * 1.5 + 0.2
    eps = torch.randn(M, pol.A, device=DEV, generator=g)
    snap = _snapshot(pol.flat)
    m32, r32 = pol.obs_rms.mean_f32.clone(), pol.obs_rms.rstd_f32.clone()
    rep = Report(f"SeptPolicy act() / critic_values(), M={M}, mode={mode}")
    note = ""
    try:
        out = pol.act(obs, eps=eps)
        values = out["values"].clone()
        torch.cuda.synchronize()
        b = pol._buf(M, False)
        P, T = b["x"], b["t"]
        check_split(rep, P, T, obs, m32, r32, E, pol.S)
        _check_self_window(rep, pol, obs, m32, r32, P, T)
        check_mlp_eval(rep, "task", pol.task, snap, T, M, top_out=P[:, :E])
        check_mlp_eval(rep, "actor", pol.actor, snap, P, M)
        check_mlp_eval(rep, "critic", pol.critic, snap, P, M)
        a, tol_a, nlp, tol_n = gaussian_sample_ref(out["mus"], eps, pol.logstd)
        check(rep, "gaussian_sample actions (fp32)", out["actions"], a, tol_a)
        check(rep, "gaussian_sample neglogp (fp32)", out["neglogpacs"], nlp, tol_n)
        again = pol.critic_values(obs)
        torch.cuda.synchronize()
        check_exact(rep, "critic_values() == act()'s values", again, values)
        check_mlp_eval(rep, "critic (critic_values)", pol.critic, snap, P, M)
        pol.task.forward(T, out=P[:, :E])            # a lone task forward: its top layer is the last launch
        torch.cuda.synchronize()
        tile = _lib.gemm_last_launch()["tile_n"]
        note = f"\n  task top layer (eval, N = {E}, into P[:, :{E}]): {tile}-wide output tile"
        if M == 16384:
            assert tile == (128 if mode == "bn128" else 256), f"task top layer at M={M} took the {tile}-wide tile"
    finally:
        print("\n" + rep.text() + note)
