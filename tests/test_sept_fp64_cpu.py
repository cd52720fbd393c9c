"""The amp_sept links of tests/test_gpu_sept_fp64.py have teeth (no GPU needed).

The SeptPolicy nets are built on the CPU (nets.MLP over a CPU FlatParams) and their kernels simulated into the same workspaces the device
fills -- bf16 operands, fp32 accumulation per 64-wide k-block, the epilogues' fp32 SiLU and bf16 roundings -- at the SEPT_SMALL widths
(E = 24, S = 22, N0 = 96) and at a mid-size one with K = 2 N0 = 1024.  The simulated composition passes the shared checkers of
tests/fp64_links.py, and each mutation below, a plausible mistake of the shared-encoder plumbing, is rejected.
"""
import pytest
import torch

from tests.fp64_links import _check_pads, _snapshot, _w, check, check_mlp, check_split
from tests.fp64_ref import UBF, BoundError, Gemm, check_exact, silu64, silu_gated, silu_gemm_tol
from tests.fp64_ref import kernel_gemm as _kernel_gemm

BF = torch.bfloat16
SMALL = dict(E=24, S=22, T=36, task_units=(40, 24), N0=96, A=11, M=160)
MID = dict(E=64, S=38, T=100, task_units=(128, 64), N0=512, A=16, M=192)


def _silu32(z):
    return z / (1.0 + torch.exp(-z))


def _silu_grad32(z):
    s = 1.0 / (1.0 + torch.exp(-z))
    return s * (1.0 + z * (1.0 - s))


class _Sim:
    """The nets of SeptPolicy on the CPU with a simulated training minibatch: split normalise, task forward into P[:, :E], actor / critic
    (one SiLU layer + head), dpre0 halves, dEmb, task backward."""

    def __init__(self, d, seed=0):
        from pulse_b200.nets import MLP, Dense, FlatParams, pad8
        self.d, E, S, T, N0, M = d, d["E"], d["S"], d["T"], d["N0"], d["M"]
        g = torch.Generator().manual_seed(seed)
        self.flat = flat = FlatParams("cpu")
        self.task = MLP(flat, T, d["task_units"], None, "silu", aug=True)
        a0, c0 = Dense(flat, E + S, N0, "silu", aug=True), Dense(flat, E + S, N0, "silu", aug=True)
        a0.ref_cols = torch.cat([torch.arange(E, E + S), torch.arange(0, E)])
        self.actor = MLP(flat, E + S, (N0,), d["A"], "silu", aug=True, first=a0)
        self.critic = MLP(flat, E + S, (N0,), 1, "silu", aug=True, first=c0)
        flat.finalize(peer=False)
        for net in (self.task, self.actor, self.critic):
            net.init_default(g)
        self.E, self.S, self.M, self.N0 = E, S, M, N0
        self.obs = torch.randn(M, S + T, generator=g) * 1.5 + 0.2
        self.mean = (torch.rand(S + T, generator=g) - 0.5) * 0.4
        self.rstd = 1.0 / torch.sqrt(torch.rand(S + T, generator=g) + 0.5)
        self.P = torch.zeros(M, self.actor.Kp0, dtype=BF)
        self.T = torch.zeros(M, self.task.Kp0, dtype=BF)
        self.dpre0 = torch.zeros(M, 2 * N0, dtype=BF)
        self.demb = torch.zeros(M, pad8(E), dtype=BF)
        self.actor.provide_dact0(M, self.dpre0[:, :N0])
        self.critic.provide_dact0(M, self.dpre0[:, N0:])
        self.dmu = torch.zeros(M, pad8(d["A"]), dtype=BF)
        self.dmu[:, :d["A"]] = (torch.randn(M, d["A"], generator=g) * 1e-2).to(BF)
        self.dv = torch.zeros(M, 8, dtype=BF)
        self.dv[:, 0] = (torch.randn(M, generator=g) * 1e-2).to(BF)
        self.g = g
        self.snap = _snapshot(flat)
        self.run()

    def normalize(self, P, T):
        """pulse_normalize_split: P[:, E:] = [self | 1 | 0...], T = [task | 1 | 0...]; P[:, :E] is left alone."""
        E, S = self.E, self.S
        y = torch.clamp((self.obs - self.mean) * self.rstd, -5.0, 5.0).to(BF)
        P[:, E:] = 0
        P[:, E:E + S] = y[:, :S]
        P[:, E + S] = 1.0
        Tn = self.obs.shape[1] - S
        T.zero_()
        T[:, :Tn] = y[:, S:]
        T[:, Tn] = 1.0

    def W(self, l):
        return _w(self.snap, self.flat, l)

    def forward(self, net, x, out=None):
        """Training forward: pre = bf16(acc), act = bf16(silu(pre)) (into `out` for the top of a headless net), fp32 head."""
        ws = net._workspace(self.M, True)
        h = x
        for i, l in enumerate(net.layers):
            acc = _kernel_gemm(h[:, :l.Kp], self.W(l).T)
            if i == len(net.layers) - 1 and not net.headless:
                ws["out"][:] = acc
                break
            pre = acc.to(BF)
            ws["pre"][i][:, :l.N] = pre
            dst = out if (out is not None and i == len(net.layers) - 1) else ws["act"][i]
            dst[:, :l.N] = _silu32(pre.float()).to(BF)
            h = dst
        ws["x"] = x

    def dgrad(self, dy, W, pre):
        return (_kernel_gemm(dy, W) * _silu_grad32(pre.float())).to(BF)

    def run(self):
        E, N0, M = self.E, self.N0, self.M
        self.normalize(self.P, self.T)
        self.forward(self.task, self.T, out=self.P[:, :E])
        self.forward(self.actor, self.P)
        self.forward(self.critic, self.P)
        for net, dout in ((self.actor, self.dmu), (self.critic, self.dv)):
            ws, head = net._ws[(M, True)], net.layers[1]
            ws["dact"][0][:, :N0] = self.dgrad(dout[:, :head.N], self.W(head)[:, :N0], ws["pre"][0][:, :N0])
        self.demb[:, :E] = self.emb_grad()
        wt = self.task._ws[(M, True)]
        t0, t1 = self.task.layers
        wt["dact"][0][:, :t0.N] = self.dgrad(self.demb[:, :E], self.W(t1)[:, :t0.N], wt["pre"][0][:, :t0.N])

    def w_cat(self):
        return torch.cat([self.W(self.actor.layers[0])[:, :self.E], self.W(self.critic.layers[0])[:, :self.E]])

    def emb_grad(self, a=None, w=None, gate=None):
        """dEmb = silu'(task top pre) * (dpre0 . [W_a0 ; W_c0][:, :E]) as the kernel computes it (arguments: mutated operands)."""
        a = self.dpre0 if a is None else a
        w = self.w_cat() if w is None else w
        gate = self.task.top_preact(self.M)[:, :self.E] if gate is None else gate
        return (_kernel_gemm(a, w) * _silu_grad32(gate.float())).to(BF)

    # ---- the links as tests/test_gpu_sept_fp64.py checks them
    def check_demb(self, demb=None):
        demb = self.demb if demb is None else demb
        y, acc = silu_gated(Gemm(self.dpre0[:, :2 * self.N0], self.w_cat()), self.task.top_preact(self.M)[:, :self.E])
        check(None, "dEmb", demb[:, :self.E], y, acc * (1 + UBF) + UBF * y.abs())
        _check_pads(None, "dEmb", demb, self.E)

    def check_split(self, P=None):
        check_split(None, self.P if P is None else P, self.T, self.obs, self.mean, self.rstd, self.E, self.S)

    def check_self_window(self, P):
        again = torch.full_like(self.P, 3.0)
        self.normalize(again, torch.zeros_like(self.T))
        check_exact(None, "self window", P[:, self.E:], again[:, self.E:])

    def check_all(self):
        self.check_split()
        self.check_self_window(self.P)
        check_mlp(None, "task", self.task, self.snap, self.T, self.demb, self.M, top_out=self.P[:, :self.E])
        check_mlp(None, "actor", self.actor, self.snap, self.P, self.dmu, self.M)
        check_mlp(None, "critic", self.critic, self.snap, self.P, self.dv, self.M)
        self.check_demb()


@pytest.fixture(scope="module", params=["small", "mid"])
def sim(request):
    return _Sim(SMALL if request.param == "small" else MID, seed=1 if request.param == "small" else 2)


def _rejects(fn):
    with pytest.raises(BoundError):
        fn()


# ---------------------------------------------------------------------------------------------------- the simulated kernels pass
def test_simulated_sept_minibatch_passes(sim):
    """Split operands, the headless task forward into P[:, :E], SiLU-gated dgrads into the dpre0 halves, dEmb, the task backward."""
    assert 2 * sim.N0 >= 1024 or sim.E == 24
    sim.check_all()


def test_simulated_eval_silu_passes(sim):
    """Eval path: the register epilogue's SiLU on the accumulator rounded to bf16 (on the fp32 one in a column group that reaches past N),
    then bf16 -- against silu64(y64) with silu_gemm_tol."""
    l = sim.actor.layers[0]
    g = Gemm(sim.P[:, :l.Kp], sim.W(l).T)
    acc = _kernel_gemm(sim.P[:, :l.Kp], sim.W(l).T)
    check(None, "eval act (silu of the bf16-rounded accumulator)", _silu32(acc.to(BF).float()).to(BF), silu64(g.y), silu_gemm_tol(g))
    check(None, "eval act (silu of the fp32 accumulator)", _silu32(acc).to(BF), silu64(g.y), silu_gemm_tol(g))


# --------------------------------------------------------------------------------------------------------- mutations are rejected
def test_rejects_demb_without_the_critic_half(sim):
    N0 = sim.N0
    _rejects(lambda: sim.check_demb(sim.emb_grad(a=sim.dpre0[:, :N0], w=sim.w_cat()[:N0])))


def test_rejects_demb_missing_the_first_k_block_of_the_critic_half(sim):
    a = sim.dpre0.clone()
    a[:, sim.N0:sim.N0 + 64] = 0
    _rejects(lambda: sim.check_demb(sim.emb_grad(a=a)))


def test_rejects_demb_reading_both_halves_from_the_actor_rows(sim):
    wa = sim.W(sim.actor.layers[0])[:, :sim.E]
    _rejects(lambda: sim.check_demb(sim.emb_grad(w=torch.cat([wa, wa]))))


def test_rejects_demb_gated_by_the_activation_instead_of_the_pre_activation(sim):
    _rejects(lambda: sim.check_demb(sim.emb_grad(gate=sim.P[:, :sim.E])))


def test_rejects_demb_gated_by_task_layer_0(sim):
    _rejects(lambda: sim.check_demb(sim.emb_grad(gate=sim.task._ws[(sim.M, True)]["pre"][0][:, :sim.E])))


def test_rejects_layer0_weights_in_the_reference_column_order(sim):
    """The kernel applies W_a0 as if P were [self | emb] (Dense.ref_cols order) instead of [emb | self]: check_mlp's layer-0 link."""
    l = sim.actor.layers[0]
    W = sim.W(l)
    Wr = W.clone()
    Wr[:, :l.K] = W[:, l.ref_cols]
    x = sim.P[:, :l.Kp]
    Gemm(x, W.T).check(None, "actor L0 pre (bf16)", _kernel_gemm(x, W.T).to(BF))
    _rejects(lambda: Gemm(x, W.T).check(None, "actor L0 pre (bf16)", _kernel_gemm(x, Wr.T).to(BF)))


@pytest.mark.parametrize("what", ["zeros", "values"])
def test_rejects_task_epilogue_writing_past_the_embedding(sim, what):
    P = sim.P.clone()
    E = sim.E
    P[:, E:E + 8] = 0 if what == "zeros" else _silu32(sim.task.top_preact(sim.M)[:, :8].float()).to(BF)
    _rejects(lambda: sim.check_self_window(P))
    _rejects(lambda: sim.check_split(P))


def test_rejects_missing_ones_column(sim):
    P = sim.P.clone()
    P[:, sim.E + sim.S] = 0
    _rejects(lambda: sim.check_split(P))


def test_rejects_weight_view_one_adam_step_stale(sim):
    """dEmb computed from the bf16 weights of one Adam step before the snapshot the reference uses (lr 2e-5, first step: lr * sign)."""
    flat = sim.flat
    stale = sim.w_cat()
    p = flat.params.clone()
    step = 2e-5 * torch.sign(torch.randn(p.shape, generator=sim.g))
    snap = dict(sim.snap, pb=(p - step).to(BF))
    fresh = torch.cat([_w(snap, flat, sim.actor.layers[0])[:, :sim.E], _w(snap, flat, sim.critic.layers[0])[:, :sim.E]])
    assert not torch.equal(fresh, stale)
    y, acc = silu_gated(Gemm(sim.dpre0, fresh), sim.task.top_preact(sim.M)[:, :sim.E])
    check(None, "dEmb (fresh weights)", sim.emb_grad(w=fresh), y, acc * (1 + UBF) + UBF * y.abs())
    _rejects(lambda: check(None, "dEmb (stale view)", sim.emb_grad(w=stale), y, acc * (1 + UBF) + UBF * y.abs()))


def test_rejects_eval_silu_on_a_bf16_accumulator_without_the_bias_column(sim):
    l = sim.actor.layers[0]
    x = sim.P[:, :l.Kp].clone()
    g = Gemm(x, sim.W(l).T)
    x[:, l.K] = 0                                           # the ones column: the bias dropped
    bad = _silu32(_kernel_gemm(x, sim.W(l).T).to(BF).float()).to(BF)
    _rejects(lambda: check(None, "eval act", bad, silu64(g.y), silu_gemm_tol(g)))
