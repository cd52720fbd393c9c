"""The evaluation pass of the two `im_amp` policies (`EvalStepsB200` over `PlayStepsB200` / `ImZStepsB200`) on a synthetic MotionLib
with a deterministic device-side stand-in for the physics: every step it sets the rigid bodies to the reference state at the step's
time, translated by an amount that grows with the episode and depends on the PD targets, so the policy decides which envs cross the
0.5 m mean distance.

Bars: exact tracking (no displacement) gives zero metrics, no termination and success rate 1 -- this pins the time of `body_pos_gt`;
the frames, recorded through the `record` hook, fed to the oracle (oracle/eval_oracle.py) give the same failed / success keys, the same
number of steps and `eval_info` within test_gpu_eval.py's tolerance, over several chunks with U not a multiple of N and over one chunk
at 16384 envs; graph and eager runs give bit-identical sums, counts, termination states and steps; the policy's weights, Adam moments
and running statistics, the driver's MotionLib and graphs are untouched and a training iteration runs after the pass; the PMCP weights
follow the oracle's failed keys."""
import numpy as np
import pytest
import torch

from tests.helpers import exact_step_inputs, exact_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VR = (13, 18, 23)
TABLE_KEYS = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa")


class SynthDataset:
    """A MotionDatasetB200 whose chunk tables are cut from synthetic tables (no forward kinematics): `load_motions` selects the clips
    exactly as MotionDatasetB200 does and builds a MotionLibB200 over their frames; the PMCP updates are MotionDatasetB200's."""

    def __init__(self, num_unique, seed, max_frames=120, spread=110):
        from pulse_b200.motion_dataset import MotionDatasetB200
        self.tb = exact_tables(num_unique, seed=seed, max_frames=max_frames, spread=spread)
        self.ds = MotionDatasetB200({f"clip_{i:05d}": {} for i in range(num_unique)}, list(range(-1, 23)), np.zeros((24, 3)), device=DEV)
        self.loads = 0

    def __getattr__(self, name):
        return getattr(self.ds, name)

    def load_motions(self, n, random_sample=True, start_idx=0, max_len=-1, eval_mode=False):
        from pulse_b200.motion_lib import MotionLibB200
        assert not random_sample and eval_mode and max_len == -1
        ids = self.ds.select(n, random_sample=False, start_idx=start_idx)
        tb = self.tb
        rows = torch.cat([torch.arange(int(tb.length_starts[i]), int(tb.length_starts[i] + tb.num_frames[i])) for i in ids.tolist()])
        nf = tb.num_frames[ids]
        t = {k: getattr(tb, k)[rows] for k in TABLE_KEYS}
        t.update(lengths=tb.lengths[ids], num_frames=nf, dt=tb.dt[ids], length_starts=torch.cumsum(nf, 0) - nf)
        self.loads += 1
        return MotionLibB200.from_tables(t, device=DEV)


def _sim(n, seed):
    """Isaac-Gym shaped simulator tensors (2 actors per env, 72 dofs, 26 bodies) and the task's training state."""
    tb = exact_tables(31, seed=seed + 100)
    z, _ = exact_step_inputs(tb, n, seed=seed)
    body = torch.zeros(n, 26, 13)
    body[:, :24] = z["body_state"]
    root = torch.zeros(n, 2, 13)
    root[:, 0] = body[:, 0]
    dof = torch.zeros(n, 72, 2)
    dof[:, :69, 0], dof[:, :69, 1] = z["dof_pos"], z["dof_vel"]
    sim = dict(body_state=body, root_all=root, dof_state=dof, progress_buf=z["progress_buf"].clone(), motion_ids=z["motion_ids"].clone(),
               motion_start_times=z["start_times"].clone(), motion_start_offset=z["start_offset"].clone(), global_offset=z["global_offset"].clone(),
               dof_force=z["dof_force"], cycle_counter=torch.zeros(n, dtype=torch.int32), contact_forces=torch.zeros(n, 26, 3),
               actor_ids=torch.arange(n, dtype=torch.int32) * 2)
    sim = {k: v.to(DEV) for k, v in sim.items()}
    sim.update(root_states=sim["root_all"][:, 0], dof_pos=sim["dof_state"][:, :69, 0], dof_vel=sim["dof_state"][:, :69, 1])
    return tb, sim


def _policy(obs, actions, seed):
    from pulse_b200.ppo import PPOPolicy
    pol = PPOPolicy(obs_size=obs, num_actions=actions, units=(256, 128), act="silu", logstd=-1.5, device=DEV, seed=seed)
    g = torch.Generator().manual_seed(seed + 40)
    pol.obs_rms.running_mean.copy_(0.1 * torch.randn(obs, generator=g, dtype=torch.float64))
    pol.obs_rms.running_var.copy_(0.5 + torch.rand(obs, generator=g, dtype=torch.float64))
    pol.obs_rms._refresh()
    return pol


def _driver(kind, n, seed=3, use_graphs=True):
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    from pulse_b200.motion_lib import MotionLibB200
    tb, sim = _sim(n, seed)
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in TABLE_KEYS + ("lengths", "num_frames", "dt", "length_starts")}, device=DEV)
    g = torch.Generator().manual_seed(seed + 1)
    pd_off, pd_scale = torch.randn(69, generator=g).to(DEV), (0.5 + torch.rand(69, generator=g)).to(DEV)
    if kind == "im":
        from pulse_b200.rollout import PlayStepsB200
        d = PlayStepsB200(HumanoidImCompute(ml), _policy(934, 69, seed), sim, horizon=4, pd_offset=pd_off, pd_scale=pd_scale,
                          use_graphs=use_graphs, reset_seed=5, time_steps=False)
    else:
        from pulse_b200.imz_rollout import ImZStepsB200
        from pulse_b200.vae import PulseVAE
        comp = HumanoidImCompute(ml, ImConfig(reset_body_ids=VR, track_body_ids=VR))
        freeze = torch.zeros(69, dtype=torch.uint8)
        freeze[[9, 10, 11, 66, 67, 68]] = 1
        d = ImZStepsB200(comp, _policy(comp.obs_size, 32, seed), PulseVAE(device=DEV, with_critic=False, seed=1), sim, horizon=4,
                         pd_offset=pd_off, pd_scale=pd_scale, pd_freeze=freeze.to(DEV), use_graphs=use_graphs, reset_seed=5)
    d.first_observation()
    return d


def _physics(ev, rate):
    """The stand-in physics: bodies = the reference at (progress + 1) dt + start + offset (the time the step kernel and `body_pos_gt`
    read after progress += 1), all translated by rate * (progress + 1) * w along a PD-target direction, w in (0, 1) the standardised
    mean of six PD targets through a sigmoid."""
    def physics(t):
        body = ev.sim["body_state"]
        times = (ev.progress_buf + 1) * ev.cfg.dt + ev.motion_start_times + ev.motion_start_offset
        ms = ev.comp.motion_lib.get_motion_state(ev.motion_ids, times, offset=ev.global_offset)
        pos = ms["rg_pos"]
        if rate:
            p = ev.pd_tar
            direction = p[:, 0:3] / (p[:, 0:3].norm(dim=-1, keepdim=True) + 1e-3)
            m = p[:, 3:9].mean(-1, keepdim=True)
            w = torch.sigmoid(2.0 * (m - m.mean()) / (m.std() + 1e-6))           # in (0, 1), spread over the envs by the policy's output
            pos = pos + (rate * (ev.progress_buf + 1).unsqueeze(-1).float() * w * direction).unsqueeze(1)
        body[:, :24] = torch.cat([pos, ms["rb_rot"], ms["body_vel"], ms["body_ang_vel"]], dim=-1)
    return physics


def _eval(d, ds, rate=None, record=False, pmcp=None, **kw):
    from pulse_b200.evaluation import EvalStepsB200
    ev = EvalStepsB200(d, **kw)
    if rate is not None:
        ev.physics = _physics(ev, rate)
    chunks = []
    if record:
        load = ev._load_chunk

        def load_chunk(start_idx):
            num_steps, ids = load(start_idx)
            chunks.append({"num_steps": num_steps, "ids": ids, "frames": []})
            return num_steps, ids
        ev._load_chunk = load_chunk
        ev.record = lambda pos, gt, term: chunks[-1]["frames"].append((pos.cpu().numpy(), gt.cpu().numpy(), term.cpu().numpy().astype(bool)))
    out = ev.run(ds, **(pmcp or {}))
    return ev, out, chunks


def _oracle(chunks, N, U, keys):
    from oracle.eval_oracle import EvalOracle
    orc = EvalOracle(N, U, keys)
    steps = 0
    for c in chunks:
        for pos, gt, term in c["frames"]:
            done, end, info = orc.post_step(term, np.linalg.norm(pos - gt, axis=-1).mean(-1), pos, gt, c["num_steps"], c["ids"])
            steps += 1
            if done or end:
                break
        else:
            raise AssertionError("the recorded frames of a chunk end before the oracle ends it")
    assert end
    return info, steps


# ------------------------------------------------------------------------------------------------ exact tracking
@pytest.mark.parametrize("kind", ["im", "imz"])
def test_exact_tracking_gives_zero_metrics(kind):
    N, U = 64, 150
    d = _driver(kind, N)
    ds = SynthDataset(U, seed=7)
    _, out, _ = _eval(d, ds, rate=0.0)
    info = out["eval_info"]
    assert out["chunks"] == 3 and ds.loads == 3
    assert info["eval_success_rate"] == 1.0 and len(out["failed_keys"]) == 0 and len(out["success_keys"]) == U
    for k in ("eval_mpjpe_all", "eval_mpjpe_succ", "mpjpel_all", "mpjpel_succ", "vel_dist", "accel_dist"):
        assert info[k] == 0.0, (k, info[k])
    assert abs(info["mpjpe_pa"]) < 1e-3, info["mpjpe_pa"]


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("kind,N,U,rate,max_frames", [("im", 64, 150, 0.02, 120), ("imz", 64, 150, 0.02, 120),
                                                      ("im", 16384, 3000, 0.03, 40), ("imz", 16384, 3000, 0.03, 40)])
def test_pass_matches_oracle(kind, N, U, rate, max_frames):
    d = _driver(kind, N)
    ds = SynthDataset(U, seed=11, max_frames=max_frames, spread=max_frames - 5)
    _, out, chunks = _eval(d, ds, rate=rate, record=True)
    info, steps = _oracle(chunks, N, U, ds._motion_data_keys)
    assert out["chunks"] == len(chunks) == -(-U // N)
    assert out["steps"] == steps
    failed = sorted(np.asarray(info["failed_keys"]).tolist())
    assert sorted(out["failed_keys"].tolist()) == failed
    assert sorted(out["success_keys"].tolist()) == sorted(np.asarray(info["success_keys"]).tolist())
    assert 0 < len(failed) < U                                                     # the policy's PD targets decide: some fail, some do not
    for k, v in info["eval_info"].items():
        got = out["eval_info"][k]
        assert abs(got - v) <= 2e-4 * max(1.0, abs(v)), (k, got, v)


# ------------------------------------------------------------------------------------------------ graph against eager
@pytest.mark.parametrize("kind,rate", [("im", None), ("im", 0.02), ("imz", None), ("imz", 0.02)])
def test_graph_equals_eager(kind, rate):
    N, U = 64, 150
    runs = []
    for graphs in (True, False):
        d = _driver(kind, N)
        ev, out, _ = _eval(d, SynthDataset(U, seed=13), rate=rate, use_graphs=graphs)
        runs.append(out)
    a, b = runs
    assert a["steps"] == b["steps"] and np.array_equal(a["terminated"], b["terminated"])
    assert np.array_equal(a["per_sequence"]["sums"], b["per_sequence"]["sums"])
    assert np.array_equal(a["per_sequence"]["counts"], b["per_sequence"]["counts"])


# ------------------------------------------------------------------------------------------------ isolation and PMCP
def _snapshot(d):
    pol = d.policy
    f = pol.flat
    out = {"params": f.params, "exp_avg": f.exp_avg, "exp_avg_sq": f.exp_avg_sq, "step": f.step, "logstd": pol.logstd}
    for name, rms in (("obs", pol.obs_rms), ("value", pol.value_rms), ("disc", getattr(pol.disc, "rms", None) if pol.disc is not None else None)):
        if rms is not None:
            out.update({f"{name}_mean": rms.running_mean, f"{name}_var": rms.running_var, f"{name}_count": rms.count})
    if getattr(d, "vae", None) is not None:
        out.update(vae_mean=d.vae.obs_rms.running_mean, vae_var=d.vae.obs_rms.running_var)
    return {k: v.clone() for k, v in out.items()}


@pytest.mark.parametrize("kind", ["im", "imz"])
def test_pass_leaves_training_state_and_graphs(kind):
    N, U = 64, 150
    d = _driver(kind, N)
    def iteration():
        d.play_steps()
        d.finish()
        if kind == "imz":
            d.train_epoch(mini_epochs=1, minibatch=N * d.T)
    for _ in range(2):                                      # eager, then captured: the driver's graphs exist before the pass
        iteration()
    torch.cuda.synchronize()
    before, lib, graphs = _snapshot(d), d.comp.motion_lib, dict(d._graphs)
    ds = SynthDataset(U, seed=17)
    d.evaluate(ds, auto_pmcp_soft=True)                                      # one K-step graph per poll
    d.evaluate(ds, physics=lambda t: _physics(d.eval_steps, 0.02)(t), auto_pmcp_soft=True)   # graph segments around the hook
    torch.cuda.synchronize()
    after = _snapshot(d)
    for k in before:
        assert torch.equal(before[k], after[k]), k
    assert d.comp.motion_lib is lib and d.comp.cfg.termination_distance == 0.25 and not d.comp.cfg.use_mean_reset
    assert d._graphs == graphs                                                # same keys, same graph objects
    assert int(d.reset_buf.sum()) == 0 and int(d.sim["progress_buf"].sum()) == 0   # every env reset into training
    for _ in range(2):
        iteration()
    torch.cuda.synchronize()
    assert d._graphs.keys() == graphs.keys() and all(d._graphs[k] is graphs[k] for k in graphs)   # replayed, not captured again
    assert bool(torch.isfinite(d.obses).all()) and bool(torch.isfinite(d.adv).all())


@pytest.mark.parametrize("kind,soft", [("im", True), ("imz", True), ("im", False)])
def test_pmcp_weights_follow_oracle_failed_keys(kind, soft):
    from pulse_b200.motion_dataset import MotionDatasetB200
    N, U = 64, 150
    d = _driver(kind, N)
    ds = SynthDataset(U, seed=19)
    ds.ds._termination_history[::9] = 2.0                   # an earlier pass's failure counts
    hist0 = ds.ds._termination_history.clone()
    _, out, chunks = _eval(d, ds, rate=0.02, record=True, pmcp={"auto_pmcp": not soft, "auto_pmcp_soft": soft})
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
