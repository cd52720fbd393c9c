"""The rollout references of tests/test_gpu_rollout_fp64.py have teeth (no GPU needed).

Each reference added for the rollout side -- policy_post_ref, philox_normals_ref, pnn_compose_ref, reparam_ref, gae_ref,
adv_normalize_ref -- and check_mlp_eval's head1 GEMV and strided-slice head run here against an fp32 CPU simulation of the kernel they
check, which must pass, and against mutated simulations, plausible mistakes of those kernels, which must fail with the link named.
"""
import math

import numpy as np
import pytest
import torch

from tests.fp64_links import _snapshot, _w, check_mlp_eval
from tests.fp64_ref import (U32, BoundError, adv_normalize_ref, check, check_exact, gae_ref, kernel_gemm, latent_post_ref, philox_pair_normals,
                            pnn_compose_ref, policy_post_ref, reparam_ref)
from tests.philox_ref import philox4x32_10

BF = torch.bfloat16
F32 = np.float32


def _rejects(fn, link):
    with pytest.raises(BoundError, match=link):
        fn()


# ------------------------------------------------------------------------------------------------------------------ policy_post
def _policy_post_sim(mu, eps, logstd, value, vmean, vvar, veps=1e-5, drop_logstd=False, no_clamp=False):
    """policy_post_kernel in fp32: a = mu + expf(l) e, z = (a - mu) / sigma, neglogp = 0.5 sum z^2 + 0.5f log(2 pi)f A + sum l; the
    value de-normalisation of value_unnorm.cuh."""
    A = mu.shape[1]
    sg = torch.exp(logstd)
    a = mu + sg * eps
    z = (a - mu) / sg
    acc = (z * z).sum(-1)
    ls = logstd.sum()
    nlp = 0.5 * acc + F32(0.5) * F32(1.8378770664093453) * A
    if not drop_logstd:
        nlp = nlp + ls
    y = value if no_clamp else torch.clamp(value, -5.0, 5.0)
    sd = torch.sqrt(vvar.float() + F32(veps))
    return a, nlp, y * sd + vmean.float()


@pytest.fixture(scope="module")
def post():
    g = torch.Generator().manual_seed(3)
    M, A = 512, 69
    mu = torch.randn(M, A, generator=g) * 0.5
    eps = torch.randn(M, A, generator=g)
    logstd = torch.full((A,), -2.9)
    value = torch.randn(M, 1, generator=g) * 2 + 5.0          # about half the rows past the clamp
    vmean, vvar = torch.tensor([0.7], dtype=torch.float64), torch.tensor([2.3], dtype=torch.float64)
    return mu, eps, logstd, value, vmean, vvar


def _check_post(post, a, nlp, v):
    mu, eps, logstd, value, vmean, vvar = post
    ref = policy_post_ref(mu, eps, logstd, value=value, value_mean=vmean, value_var=vvar)
    check(None, "actions", a, *ref["actions"])
    check(None, "neglogp", nlp, *ref["neglogp"])
    check(None, "values (value_unnorm)", v, *ref["values"])


def test_simulated_policy_post_passes(post):
    _check_post(post, *_policy_post_sim(*post))


def test_rejects_neglogp_without_the_logstd_term(post):
    _rejects(lambda: _check_post(post, *_policy_post_sim(*post, drop_logstd=True)), "neglogp")


def test_rejects_value_unnorm_without_its_clamp(post):
    _rejects(lambda: _check_post(post, *_policy_post_sim(*post, no_clamp=True)), "values")


# ---------------------------------------------------------------------------------------------------------------- Philox normals
def _box_muller32(seed, rows, width, offset, stride=64):
    """philox.cuh's draws in fp32 numpy: u1, u2 on the 2^-24 grid, sqrtf(-2 logf(u1)), sincosf(2 pi_f32 u2); pairs (2p, 2p + 1) from block
    (seed, row * stride + p, offset)."""
    pairs = (width + 1) // 2
    idx = (np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(stride) + np.arange(pairs, dtype=np.uint64)[None, :]).reshape(-1)
    x, y, _, _ = philox4x32_10(seed, idx, offset)
    u1 = ((x >> np.uint64(8)).astype(F32) + F32(1.0)) * F32(1.0 / 16777216.0)
    u2 = (y >> np.uint64(8)).astype(F32) * F32(1.0 / 16777216.0)
    r = np.sqrt(F32(-2.0) * np.log(u1).astype(F32)).astype(F32)
    arg = (F32(2 * math.pi) * u2).astype(F32)
    n = np.stack([r * np.cos(arg).astype(F32), r * np.sin(arg).astype(F32)], -1).reshape(rows, 2 * pairs)[:, :width]
    return torch.from_numpy(np.ascontiguousarray(n, dtype=F32))


SEED = 0x243F6A8885A308D3


def test_simulated_philox_normals_pass():
    for width in (69, 32):
        n, t = philox_pair_normals(SEED, 300, width, 1003)
        check(None, "philox draws", _box_muller32(SEED, 300, width, 1003), n, t)


def test_philox_tolerance_stays_far_below_one():
    """Near 1e-6 almost everywhere; largest where u1 -> 1 (r -> 0, where the root magnifies __logf's absolute error)."""
    _, t = philox_pair_normals(SEED, 300, 69, 7)
    assert float(t.max()) < 1e-4 and float(t.median()) < 3e-6


def test_rejects_reparam_index_row_times_pairs():
    """The reparameterisation kernel keyed (seed, r * pairs + p) in place of (seed, r * 64 + p): every row past the first draws another
    row's noise."""
    n, t = philox_pair_normals(SEED, 300, 32, 11)
    _rejects(lambda: check(None, "philox draws", _box_muller32(SEED, 300, 32, 11, stride=16), n, t), "philox draws")


def test_rejects_philox_offset_off_by_one():
    n, t = philox_pair_normals(SEED, 64, 69, 11)
    _rejects(lambda: check(None, "philox draws", _box_muller32(SEED, 64, 69, 12), n, t), "philox draws")


# ----------------------------------------------------------------------------------------------------------------- pnn_compose
def _compose_sim(w, acts, act, skip_last=False):
    K = w.shape[1] - (1 if skip_last else 0)
    s = torch.zeros(acts.shape[1:])
    for k in range(K):
        wk = w[:, k:k + 1]
        if act == "silu":
            wk = wk / (1.0 + torch.exp(-wk))
        elif act == "relu":
            wk = torch.relu(wk)
        s = (wk.double() * acts[k].double() + s.double()).float()        # fmaf: one rounding
    return s


@pytest.mark.parametrize("act", ["silu", "relu", None])
def test_simulated_pnn_compose_passes_and_rejects_a_skipped_primitive(act):
    g = torch.Generator().manual_seed(5)
    w = torch.randn(300, 3, generator=g)
    acts = torch.randn(3, 300, 69, generator=g) * 0.4
    y, tol = pnn_compose_ref(w, acts, act)
    check(None, "pnn_compose", _compose_sim(w, acts, act), y, tol)
    _rejects(lambda: check(None, "pnn_compose", _compose_sim(w, acts, act, skip_last=True), y, tol), "pnn_compose")


# --------------------------------------------------------------------------------------------------------------------- reparam
def _reparam_sim(head, noise, E, mode, clamp=True, lo=-5.0, hi=2.0):
    mu = head[:, :E]
    if mode == "mean":
        return mu.to(BF)
    if mode == "residual":
        return (mu + noise).to(BF)
    lv = head[:, E:2 * E]
    if clamp:
        lv = torch.clamp(lv, lo, hi)
    return (mu + torch.exp(F32(0.5) * lv) * noise).to(BF)


@pytest.fixture(scope="module")
def rep_in():
    g = torch.Generator().manual_seed(9)
    M, E = 400, 32
    head = torch.randn(M, 2 * E, generator=g)
    head[:, E:] = torch.randn(M, E, generator=g) * 4          # log-variances on both sides of [-5, 2]
    noise = _box_muller32(SEED, M, E, 5)
    n, nt = philox_pair_normals(SEED, M, E, 5)
    return head, noise, n, nt, E


@pytest.mark.parametrize("mode", ["sample", "mean", "residual"])
def test_simulated_reparam_passes(rep_in, mode):
    head, noise, n, nt, E = rep_in
    z, tol = reparam_ref(head, n, mode, E, noise_tol=nt)
    check(None, f"reparam z ({mode})", _reparam_sim(head, noise, E, mode), z, tol)


def test_rejects_reparam_without_the_clamp(rep_in):
    head, noise, n, nt, E = rep_in
    z, tol = reparam_ref(head, n, "sample", E, noise_tol=nt)
    _rejects(lambda: check(None, "reparam z", _reparam_sim(head, noise, E, "sample", clamp=False), z, tol), "reparam z")


def test_rejects_reparam_with_the_wrong_philox_index(rep_in):
    head, _, n, nt, E = rep_in
    z, tol = reparam_ref(head, n, "sample", E, noise_tol=nt)
    wrong = _box_muller32(SEED, head.shape[0], E, 5, stride=(E + 1) // 2)
    _rejects(lambda: check(None, "reparam z", _reparam_sim(head, wrong, E, "sample"), z, tol), "reparam z")


# ------------------------------------------------------------------------------------------------------------------------- GAE
def _gae_sim(r, v, nv, d, gamma, tau, shifted_dones=False, tau_late=False):
    """gae_kernel in fp32.  shifted_dones: reads fdones[t + 1] (0 past the end); tau_late: gamma tau applied to the step after."""
    T, N = r.shape
    g, ta = F32(gamma), F32(tau)
    c = torch.tensor(g * ta, dtype=torch.float32)
    last = torch.zeros(N)
    adv, ret = torch.zeros(T, N), torch.zeros(T, N)
    for t in range(T - 1, -1, -1):
        dd = (d[t + 1] if t + 1 < T else torch.zeros(N)) if shifted_dones else d[t]
        delta = (r[t] + g * nv[t]) - v[t]
        cf = torch.tensor(g, dtype=torch.float32) if (tau_late and t == T - 2) else c
        last = delta + (cf * (1.0 - dd)) * last
        adv[t], ret[t] = last, last + v[t]
    return adv, ret


@pytest.fixture(scope="module", params=[(1, 5), (17, 257), (64, 33)])
def gae_in(request):
    T, N = request.param
    g = torch.Generator().manual_seed(T * 1000 + N)
    r = torch.randn(T, N, generator=g) * 10
    r[:, ::7] *= 100
    v = torch.randn(T, N, generator=g) * 3 + 1
    nv = torch.randn(T, N, generator=g) * 3 + 1
    d = (torch.rand(T, N, generator=g) < 0.2).float()
    d[:, 1::5] = 1.0
    return r, v, nv, d


def _check_gae(gae_in, adv, ret):
    a64, ta, r64, tr = gae_ref(*gae_in, 0.99, 0.95)
    check(None, "GAE advantages", adv, a64, ta)
    check(None, "GAE returns", ret, r64, tr)


def test_simulated_gae_passes(gae_in):
    _check_gae(gae_in, *_gae_sim(*gae_in, 0.99, 0.95))


def test_gae_bound_scales_with_the_rewards(gae_in):
    """Above a fixed 1e-6 where |r| ~ 1e3 (the fp32 error there is larger), yet a few u32 per step of the largest discounted sum."""
    r, v, nv, _ = gae_in
    T = r.shape[0]
    a64, ta, _, _ = gae_ref(*gae_in, 0.99, 0.95)
    assert float(ta.max()) > 1e-6
    scale = float(r.abs().max() + v.abs().max() + nv.abs().max()) * min(T, 1 / (1 - 0.99 * 0.95))
    assert float(ta.max()) < 16 * U32 * T * scale


def test_rejects_gae_reading_the_next_steps_done(gae_in):
    if gae_in[0].shape[0] == 1:
        pytest.skip("one step: there is no next done")
    _rejects(lambda: _check_gae(gae_in, *_gae_sim(*gae_in, 0.99, 0.95, shifted_dones=True)), "GAE advantages")


def test_rejects_gae_with_tau_dropped_on_one_step(gae_in):
    if gae_in[0].shape[0] == 1:
        pytest.skip("one step: nothing is carried")
    _rejects(lambda: _check_gae(gae_in, *_gae_sim(*gae_in, 0.99, 0.95, tau_late=True)), "GAE advantages")


def _normalize_sim(adv, biased=False):
    a = adv.double()
    n = a.numel()
    mean = a.sum() / n
    var = (((a * a).sum() - n * mean * mean) / (n if biased else n - 1)).clamp_min(0.0)
    return (adv - mean.float()) / (torch.sqrt(var).float() + F32(1e-8))


def test_simulated_advantage_normalisation_passes_and_rejects_the_biased_variance(gae_in):
    adv, _ = _gae_sim(*gae_in, 0.99, 0.95)
    flat = adv.T.reshape(-1)
    y, tol = adv_normalize_ref(flat)
    check(None, "normalised advantages", _normalize_sim(flat), y, tol)
    _rejects(lambda: check(None, "normalised advantages", _normalize_sim(flat, biased=True), y, tol), "normalised advantages")


# ---------------------------------------------------------------------------------------------------- check_mlp_eval: head1 and slices
class _Critic:
    """A bias-augmented ReLU net with a single-output head on the CPU (the imitation critic's shape at small widths), its eval workspace
    filled by simulated kernels: bf16 ReLU layers, the head1 GEMV (8-column chunks, fp32 fma) into ws['out'] or a strided slice."""

    def __init__(self, K=93, units=(192, 136), M=160, head=1, seed=0):
        from pulse_b200.nets import MLP, FlatParams
        g = torch.Generator().manual_seed(seed)
        self.flat = FlatParams("cpu")
        self.mlp = MLP(self.flat, K, units, head, "relu", aug=True)
        self.flat.finalize(peer=False)
        self.mlp.init_default(g)
        self.snap = _snapshot(self.flat)
        self.M, self.K = M, K
        x = torch.zeros(M, self.mlp.Kp0, dtype=BF)
        x[:, :K] = torch.randn(M, K, generator=g).to(BF)
        x[:, K] = 1.0
        self.x = x

    def run(self, out=None, skip_chunk=None):
        ws = self.mlp._workspace(self.M, False)
        h = self.x
        L = self.mlp.layers
        for i, l in enumerate(L[:-1]):
            ws["act"][i][:, :l.N] = torch.relu(kernel_gemm(h[:, :l.Kp], _w(self.snap, self.flat, l).T)).to(BF)
            h = ws["act"][i]
        top = L[-1]
        w = _w(self.snap, self.flat, top)
        dst = ws["out"] if out is None else out
        if self.mlp._head1(len(L) - 1):
            acc = torch.zeros(self.M, dtype=torch.float64)
            for k0 in range(0, top.Kp, 8):
                if skip_chunk is not None and k0 == skip_chunk:
                    continue
                acc = (acc + (h[:, k0:k0 + 8].double() * w[0, k0:k0 + 8].double()).sum(-1)).float().double()
            dst[:, 0] = acc.float()
        else:
            dst[:, :top.N] = kernel_gemm(h[:, :top.Kp], w.T)
        return dst


def test_simulated_head1_gemv_passes():
    c = _Critic()
    assert c.mlp._head1(2)
    c.run()
    check_mlp_eval(None, "critic", c.mlp, c.snap, c.x, c.M)


def test_rejects_head1_gemv_skipping_the_chunk_with_the_bias_column():
    """A GEMV loop that stops one 8-column chunk early: the last chunk holding data is the one with the ones / bias column."""
    c = _Critic()
    top = c.mlp.layers[-1]
    c.run(skip_chunk=(top.K // 8) * 8)
    _rejects(lambda: check_mlp_eval(None, "critic", c.mlp, c.snap, c.x, c.M), "head1 GEMV")


def test_rejects_head1_gemv_skipping_a_middle_chunk():
    c = _Critic()
    c.run(skip_chunk=64)
    _rejects(lambda: check_mlp_eval(None, "critic", c.mlp, c.snap, c.x, c.M), "head1 GEMV")


def test_head_in_a_strided_slice_is_read_from_the_slice():
    """A headed net whose forward(out=) wrote an [M, T, A] slice: check_mlp_eval(top_out=) reads the slice; the workspace head is not
    what the kernel wrote."""
    c = _Critic(head=11, seed=1)
    buf = torch.full((c.M, 4, 11), 7.0)
    c.run(out=buf[:, 2])
    c.mlp._ws[(c.M, False)]["out"].fill_(0.0)
    check_mlp_eval(None, "actor", c.mlp, c.snap, c.x, c.M, top_out=buf[:, 2])
    _rejects(lambda: check_mlp_eval(None, "actor", c.mlp, c.snap, c.x, c.M, top_out=buf[:, 1]), "in the slice")
    _rejects(lambda: check_mlp_eval(None, "actor", c.mlp, c.snap, c.x, c.M), "eval head")


# ------------------------------------------------------------------------------------------------------------------- latent_post
def test_simulated_latent_post_passes_and_rejects_prior_plus_mu(post):
    """latent_post_kernel: policy_post_kernel's arithmetic at A = 32, then z = bf16(fp32(prior_mu + a)).  A kernel writing prior_mu + mu
    (the mean instead of the sampled action) fails the exact z link."""
    mu, eps, logstd, value, vmean, vvar = post
    mu, eps, logstd = mu[:, :32].contiguous(), eps[:, :32].contiguous(), logstd[:32]
    prior = torch.randn(mu.shape[0], 64, generator=torch.Generator().manual_seed(4))
    a, nlp, v = _policy_post_sim(mu, eps, logstd, value, vmean, vvar)
    ref = latent_post_ref(mu, eps, logstd, prior[:, :32], a, value=value, value_mean=vmean, value_var=vvar)
    check(None, "latent_post actions", a, *ref["actions"])
    check(None, "latent_post neglogp", nlp, *ref["neglogp"])
    check(None, "latent_post values", v, *ref["values"])
    check_exact(None, "latent_post z", (prior[:, :32] + a).to(BF), ref["z"])
    _rejects(lambda: check_exact(None, "latent_post z", (prior[:, :32] + mu).to(BF), ref["z"]), "latent_post z")
