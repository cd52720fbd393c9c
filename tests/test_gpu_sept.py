"""amp_sept policy (pedestrian terrain task) on the GPU: split normalisation kernel, SeptPolicy against the reference-generated fixture
(tests/golden/sept.npz) and the oracle's fp32 autograd at production size, checkpoint / optimizer-state keys, determinism, and the agent mixin.

Tolerances as tests/test_gpu_ppo.py: GEMMs run bf16 x bf16 -> fp32, so outputs within 2e-2, losses within 1e-3 and gradients compared
by cosine similarity.  The actor and critic losses are compared with the reference's formulas evaluated on the device's own mu / value: with
sigma = exp(-1) the probability ratio exp(old - new) of 32 actions amplifies the 2e-2 bf16 output tolerance to several percent of the
actor loss, so comparing them with the fp32 reference's outputs would test the bf16 rounding, not the loss."""
import pytest
import torch

from tests.helpers import load_npz
from tests.sept_fixture import SEPT_FULL, SEPT_SMALL, normalise, sept_fixture

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _policy(d, seed=0, load=True):
    from pulse_b200.sept import SeptPolicy
    pol = SeptPolicy(self_obs_size=d["S"], task_obs_size_detail={"traj": d["traj"], "heightmap": d["heightmap"]}, task_units=d["task_units"],
                     units=d["units"], act="silu", num_actions=d["A"], with_disc=True, amp_obs_size=d["amp"], disc_units=d["disc_units"], device=DEV,
                     seed=seed)
    sd, b, chk = sept_fixture(d)
    if load:
        full = {"a2c_network." + k: v for k, v in sd.items()}
        full.update({"running_mean_std.running_mean": b["obs_mean"].double(), "running_mean_std.running_var": b["obs_var"].double(),
                     "amp_input_mean_std.running_mean": b["amp_mean"].double(), "amp_input_mean_std.running_var": b["amp_var"].double()})
        pol.load_state_dict(full)
    # the fixture normalises all three AMP batches with the same statistics (eval mode); in training mode the normaliser would merge the
    # agent batch before normalising the replay batch
    pol.disc.rms.frozen = True
    return pol, sd, {k: v.to(DEV) for k, v in b.items()}, chk


def _device_grads(pol):
    out = {}
    for name, l in pol._named_layers():
        n = name[len("a2c_network."):]
        out[n + ".weight"], out[n + ".bias"] = l.ref_weight("grads"), l.bias_grad.clone()
    return out


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.double().flatten(), b.double().flatten().to(a.device), dim=0).item()


def _own_losses(pol, out, b, old):
    """the reference's PPO loss terms (oracle/pulse_oracle.py) on the device's own act() outputs"""
    from oracle import pulse_oracle as po
    value = pol.value_rms.normalize_values(out["values"])          # back to the critic's raw output (the normaliser is at its identity)
    return po.ppo_total_loss(out["mus"], value[:, 0], old, b["advantages"], b["returns"], b["actions"], pol.logstd)


def _train(pol, b, old_nlp, **kw):
    amp = tuple(b[k] for k in ("amp_agent", "amp_replay", "amp_demo"))
    return pol.train_minibatch(b["obs"], b["actions"], old_nlp, b["advantages"], b["returns"], amp=amp, **kw)


# ---------------------------------------------------------------------------------------------------------------- 1. split normalise
@pytest.mark.parametrize("M", [1, 7, 1000, 16384])
def test_normalize_split_equals_normalize_moments(M):
    """pulse_normalize_split == pulse_normalize_moments on the same rows, rearranged: bf16 columns bit-identical, ones / padding exact,
    fp64 moments within 1e-12; the eval variant (sums = NULL) writes no moments."""
    from pulse_b200 import _lib
    lib, st = _lib.load(), _lib.current_stream(DEV)
    S, T, E = 358, 1044, 256
    g = torch.Generator(device=DEV).manual_seed(M)
    x = torch.randn(M, S + T, device=DEV, generator=g) * 2 + 0.5
    mean = torch.linspace(-0.5, 0.5, S + T, device=DEV)
    rstd = 1.0 / torch.sqrt(torch.linspace(0.5, 2.0, S + T, device=DEV) + 1e-5)
    ref, ref_sums = torch.zeros(M, 1408, device=DEV, dtype=torch.bfloat16), torch.zeros(2 * (S + T), device=DEV, dtype=torch.float64)
    _lib.check(lib.pulse_normalize_moments(x.data_ptr(), x.stride(0), M, S + T, mean.data_ptr(), rstd.data_ptr(), ref.data_ptr(), ref.stride(0),
                                           ref_sums.data_ptr(), 1.0, st), "pulse_normalize_moments")

    def split(sums):
        P = torch.full((M, 640), 3.0, device=DEV, dtype=torch.bfloat16)
        Tb = torch.full((M, 1088), 3.0, device=DEV, dtype=torch.bfloat16)
        _lib.check(lib.pulse_normalize_split(x.data_ptr(), x.stride(0), M, S + T, S, mean.data_ptr(), rstd.data_ptr(), P.data_ptr(), P.stride(0), E,
                                             Tb.data_ptr(), Tb.stride(0), _lib.ptr(sums), st), "pulse_normalize_split")
        return P, Tb

    sums = torch.zeros_like(ref_sums)
    for P, Tb in (split(sums), split(None)):
        assert torch.equal(P[:, E:E + S], ref[:, :S]) and torch.equal(Tb[:, :T], ref[:, S:S + T])
        assert torch.all(P[:, :E] == 3.0)                # the embedding window is left to the task net's GEMM
        assert torch.all(P[:, E + S] == 1.0) and torch.all(P[:, E + S + 1:] == 0) and torch.all(Tb[:, T] == 1.0) and torch.all(Tb[:, T + 1:] == 0)
    torch.testing.assert_close(sums, ref_sums, atol=1e-12, rtol=1e-12)


# ---------------------------------------------------------------------------------------------------------------- 2. reference fixture
@pytest.mark.parametrize("tag,d", [("a_", SEPT_SMALL), ("b_", SEPT_FULL)])
def test_policy_matches_reference_fixture(tag, d):
    g = load_npz("sept.npz")
    pol, sd, b, chk = _policy(d)
    assert abs(chk - float(g[tag + "checksum"])) < 1e-9 * abs(chk)
    M, B = d["M"], d["B"]
    out = pol.act(b["obs"], eps=torch.zeros(M, d["A"], device=DEV))
    n = g[tag + "mu"].shape[0]
    torch.testing.assert_close(out["mus"][:n].cpu(), g[tag + "mu"], atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(out["values"][:n].cpu(), g[tag + "value"], atol=2e-2, rtol=2e-2)   # value normaliser at its identity init
    torch.testing.assert_close(pol.critic_values(b["obs"]), out["values"], atol=0, rtol=0)
    old = g[tag + "old_neglogp"].to(DEV)
    own = _own_losses(pol, out, b, old)
    stats = _train(pol, b, old, update_obs_rms=False, keep_grads=True).cpu() / M
    losses = {"a_loss": stats[0].item(), "c_loss": stats[1].item(), "b_loss": stats[2].item(), "disc_loss": pol.disc.loss_tensors(B)["disc_loss"].item()}
    refs = {"a_loss": own["a_loss"].item(), "c_loss": own["c_loss"].item(), "b_loss": float(g[tag + "b_loss"]), "disc_loss": float(g[tag + "disc_loss"])}
    for k, v in losses.items():
        assert abs(v - refs[k]) < 1e-3 * max(1.0, abs(refs[k])), (k, v, refs[k])
    grads = _device_grads(pol)
    from tests.test_sept_cpu import param_names
    names = param_names(g, tag)
    assert sorted(names) == sorted(grads)
    for nme in names:
        # the actor loss's gradient carries each row's probability ratio, which the bf16 mu moves by several percent (see the module
        # docstring); over this fixture's <= 96 rows that does not average out, in the actor and in the shared task encoder it feeds.
        # test_production_minibatch_matches_oracle_autograd holds every gradient, these included, to 0.995 at 16384 rows.
        actor = nme.startswith(("actor_mlp.", "mu.", "_task_mlp."))
        if tag == "a_":
            c = _cos(grads[nme], g[tag + "grad." + nme])
            assert c > (0.97 if actor else 0.995), (nme, c)
        else:
            gr = grads[nme]
            rel = abs(gr.double().norm().item() - float(g[tag + "gnorm." + nme])) / float(g[tag + "gnorm." + nme])
            c = _cos(gr.reshape(gr.shape[0], -1)[0] if gr.dim() > 1 else gr, g[tag + "grow0." + nme])
            assert (rel < 0.1) if actor else (rel < 0.05 and c > 0.99), (nme, rel, c)   # actor path at 64 rows: norms only


# ---------------------------------------------------------------------------------------------------------------- 3. production size
def test_production_minibatch_matches_oracle_autograd():
    from oracle import sept_oracle as so
    from oracle import pulse_oracle as po
    d = SEPT_FULL
    pol, sd, _, _ = _policy(d)
    M, B = 16384, 4096
    gen = torch.Generator(device=DEV).manual_seed(5)
    S, T, A = d["S"], d["traj"] + d["heightmap"], d["A"]
    b = {"obs": torch.randn(M, S + T, device=DEV, generator=gen) * 1.5 + 0.25, "advantages": torch.randn(M, device=DEV, generator=gen),
         "returns": torch.randn(M, device=DEV, generator=gen) * 0.5,
         **{k: torch.randn(B, d["amp"], device=DEV, generator=gen) * s for k, s in (("amp_agent", 1.0), ("amp_replay", 1.2), ("amp_demo", 0.8))}}
    _, fb, _ = sept_fixture(d)
    psd = {k: v.to(DEV).requires_grad_(k != "sigma") for k, v in sd.items()}
    obs_n = normalise(b["obs"], fb["obs_mean"], fb["obs_var"])
    amp_n = [normalise(b[k], fb["amp_mean"], fb["amp_var"]) for k in ("amp_agent", "amp_replay", "amp_demo")]
    with torch.no_grad():
        mu0 = so.eval_actor(psd, obs_n, S)
    b["actions"] = (mu0 + 0.37 * torch.randn(M, A, device=DEV, generator=gen)).contiguous()
    logstd = psd["sigma"].detach()
    old = (po.gaussian_neglogp(b["actions"], mu0, torch.exp(logstd).expand_as(mu0), logstd.expand_as(mu0))
           + 0.3 * torch.randn(M, device=DEV, generator=gen)).contiguous()
    ref = so.total_loss(psd, obs_n, b["actions"], old, b["advantages"], b["returns"], amp=amp_n, self_obs_size=S)
    names = [k for k in psd if k != "sigma"]
    rgrads = dict(zip(names, torch.autograd.grad(ref["loss"], [psd[k] for k in names])))
    out = pol.act(b["obs"], eps=torch.zeros(M, A, device=DEV))
    torch.testing.assert_close(out["mus"], ref["mu"].detach(), atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(out["values"], ref["value"].detach(), atol=2e-2, rtol=2e-2)
    own = _own_losses(pol, out, b, old)
    stats = _train(pol, b, old, update_obs_rms=False, keep_grads=True).cpu() / M
    for i, k in enumerate(("a_loss", "c_loss", "b_loss")):
        r = (ref if k == "b_loss" else own)[k].item()
        assert abs(stats[i].item() - r) < 1e-3 * max(1.0, abs(r)), (k, stats[i].item(), r)
    dl = pol.disc.loss_tensors(B)["disc_loss"].item()
    assert abs(dl - ref["disc_loss"].item()) < 1e-3 * max(1.0, abs(ref["disc_loss"].item()))
    grads = _device_grads(pol)
    for n in names:
        assert _cos(grads[n], rgrads[n]) > 0.995, (n, _cos(grads[n], rgrads[n]))


# ---------------------------------------------------------------------------------------------------------------- 4. checkpoints
def test_checkpoint_and_optimizer_state_round_trip():
    d = SEPT_SMALL
    pol, sd, b, _ = _policy(d)
    g = load_npz("sept.npz")
    from tests.test_sept_cpu import param_names
    names = param_names(g, "a_")
    out = pol.state_dict()
    for n in names + ["sigma"]:
        assert torch.equal(out["a2c_network." + n].cpu(), sd[n]), n           # fp32 masters: exact round trip
    S, E = d["S"], d["task_units"][-1]
    for net in (pol.actor, pol.critic):                                          # internal [emb | self] <-> reference [self | emb]
        w = net.layers[0].weight
        assert torch.equal(w[:, 0].cpu(), sd[("actor_mlp" if net is pol.actor else "critic_mlp") + ".0.weight"][:, S])
        assert torch.equal(w[:, E].cpu(), sd[("actor_mlp" if net is pol.actor else "critic_mlp") + ".0.weight"][:, 0])
    gen = torch.Generator().manual_seed(3)
    state = {"a2c_network." + n: {"exp_avg": torch.randn(sd[n].shape, generator=gen), "exp_avg_sq": torch.rand(sd[n].shape, generator=gen),
                                  "step": torch.tensor(7.0)} for n in names}
    pol.load_optimizer_state(state)
    back = pol.optimizer_state()
    assert sorted(back) == sorted(state)
    for n in state:
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(back[n][k].cpu(), state[n][k]), (n, k)
        assert float(back[n]["step"]) == 7.0
    m = pol.flat.view(pol.actor.layers[0].w_idx, "exp_avg")
    assert torch.equal(m[:, 0].cpu(), state["a2c_network.actor_mlp.0.weight"]["exp_avg"][:, S])


# ---------------------------------------------------------------------------------------------------------------- 5. determinism
def _sequence(d, mode, n=3, capture=False):
    from pulse_b200.sept import SeptPolicy  # noqa: F401
    pol, _, b0, _ = _policy(d)
    pol.obs_rms.frozen = True                    # fp64 atomics in the statistics add in a run-dependent order; keep them out of the bits
    pol.disc.rms.frozen = True
    g = torch.Generator(device=DEV).manual_seed(9)
    M, B = d["M"], d["B"]
    batches = []
    for i in range(n):
        b = {k: (v + 0.1 * i * torch.randn(v.shape, device=DEV, generator=g)) if v.shape[0] in (M, B) else v for k, v in b0.items()}
        b["old"] = pol.act(b["obs"], eps=torch.zeros(M, d["A"], device=DEV))["neglogpacs"].clone() + 0.1
        batches.append(b)
    amp = lambda b: tuple(b[k] for k in ("amp_agent", "amp_replay", "amp_demo"))
    step = lambda i, **kw: pol.train_minibatch(batches[i]["obs"], batches[i]["actions"], batches[i]["old"], batches[i]["advantages"],
                                               batches[i]["returns"], amp=amp(batches[i]), **kw)
    if mode == "prefetch":
        pol.prepare_inputs(batches[0]["obs"], amp(batches[0]), slot=0)
        for i in range(n):
            step(i, slot=i & 1, prepared=True, prefetch=(batches[i + 1]["obs"], amp(batches[i + 1])) if i + 1 < n else None)
    elif mode == "graph":
        step(0)                                       # warm-up: workspaces, split-K choices
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step(1)
        graph.replay()
        graph.replay()
    else:
        for i in range(n):
            step(i)
    torch.cuda.synchronize()
    return pol.flat.params.clone(), pol.stats.clone()


def test_determinism_prefetch_and_graph_replay():
    d = SEPT_SMALL
    # the loss statistics are fp64 sums over rows added with atomics: their last bits depend on the order the CTAs finish
    same_stats = lambda x, y: torch.testing.assert_close(x, y, atol=1e-12, rtol=1e-12)
    a, b = _sequence(d, "inline"), _sequence(d, "inline")
    assert torch.equal(a[0], b[0])                                              # two runs: identical weights
    same_stats(a[1], b[1])
    p = _sequence(d, "prefetch")
    assert torch.equal(a[0], p[0])                                              # prefetched operands == inline (frozen statistics)
    same_stats(a[1], p[1])
    # graph: eager step(0) + two replays of step(1) == eager step(0), step(1), step(1)
    gph = _sequence(d, "graph")
    ref = _eager_0_1_1(d)
    assert torch.equal(gph[0], ref[0])
    same_stats(gph[1], ref[1])


def _eager_0_1_1(d):
    pol, _, b0, _ = _policy(d)
    pol.obs_rms.frozen = True
    pol.disc.rms.frozen = True
    g = torch.Generator(device=DEV).manual_seed(9)
    M, B = d["M"], d["B"]
    batches = []
    for i in range(3):
        b = {k: (v + 0.1 * i * torch.randn(v.shape, device=DEV, generator=g)) if v.shape[0] in (M, B) else v for k, v in b0.items()}
        b["old"] = pol.act(b["obs"], eps=torch.zeros(M, d["A"], device=DEV))["neglogpacs"].clone() + 0.1
        batches.append(b)
    for i in (0, 1, 1):
        bb = batches[i]
        pol.train_minibatch(bb["obs"], bb["actions"], bb["old"], bb["advantages"], bb["returns"], amp=(bb["amp_agent"], bb["amp_replay"], bb["amp_demo"]))
    torch.cuda.synchronize()
    return pol.flat.params.clone(), pol.stats.clone()


# ---------------------------------------------------------------------------------------------------------------- 6. agent mixin
def test_agent_mixin_builds_sept_policy_and_writes_back():
    from pulse_b200 import PulseError
    from pulse_b200.agent_mixins import AMPAgentB200Mixin
    from pulse_b200.sept import SeptPolicy
    from tests.sept_standin import SeptAgentStandin
    d = SEPT_SMALL
    sd, b, _ = sept_fixture(d)
    b = {k: v.to(DEV) for k, v in b.items()}

    class Agent(AMPAgentB200Mixin, SeptAgentStandin):
        pass

    agent = Agent(d, sd, b, DEV)
    res = agent.get_action_values({"obs": b["obs"]})
    assert isinstance(agent._pulse, SeptPolicy)
    with torch.no_grad():
        mu_ref, v_ref = agent.reference_outputs(b["obs"])
    torch.testing.assert_close(res["mus"], mu_ref, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(res["values"], v_ref, atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(agent._eval_critic({"obs": b["obs"]}), res["values"], atol=0, rtol=0)
    M, B = d["M"], d["B"]
    agent._amp_minibatch_size = B
    agent.calc_gradients({"obs": b["obs"], "actions": b["actions"], "old_logp_actions": res["neglogpacs"].clone(), "advantages": b["advantages"],
                          "returns": b["returns"], "mu": res["mus"].clone(), "amp_obs": b["amp_agent"], "amp_obs_replay": b["amp_replay"],
                          "amp_obs_demo": b["amp_demo"]})
    assert set(agent.train_result) >= {"actor_loss", "critic_loss", "b_loss", "disc_loss"}
    after = agent.get_action_values({"obs": b["obs"]})["mus"].clone()
    agent.get_weights()                                # write-back into the reference module + optimizer state
    assert len(agent.optimizer.state) > 0
    agent.set_weights(None)                            # restore -> rebuilt from the written-back modules at the next use
    again = agent.get_action_values({"obs": b["obs"]})["mus"]
    assert torch.equal(again, after)
    for detail in ({"traj": 6, "heightmap": 30, "people": 25}, {"traj": 6, "heightmap_velocity": 90}):
        bad = Agent(d, sd, b, DEV, detail=detail)
        with pytest.raises(PulseError, match="people|heightmap_velocity"):
            bad.get_action_values({"obs": b["obs"]})
