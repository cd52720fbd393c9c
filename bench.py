#!/usr/bin/env python
"""bench.py -- env-steps/s of the PULSE HumanoidIm hot path on H100 (BASELINE.json metric).

One bench "step" = one PPO iteration of BASELINE config C4 (HumanoidIm PPO, 16384 envs total,
AMASS-shaped synthetic MotionLib, horizon 32): 32 post-physics env steps (fused reward/reset/obs
kernel + AMP-obs kernel each) followed by the rollout post-processing (GAE / returns / advantage
normalisation).  Isaac Gym physics is excluded on every arm (not installable here; BASELINE.md 3.4).
`config.phases` lists exactly what runs inside the timed region and `config.not_yet` what the
reference iteration additionally does that this build does not run yet.

Contract: `python bench.py --gpus N --steps K --warmup W` (torchrun for N > 1), one JSON line on
rank 0.  `--dump-outputs DIR` writes what the last timed iteration computed as DIR/<name>.npy (seeded inputs: two builds
run with the same arguments can be compared output for output).  `--impl reference` times the CPU port of the reference path (oracle/, kind "port") on the
host cores.  Envs shard across ranks (16384 / N each, "strong" scaling); no data-path collective in
the rollout; NCCL is only used for the timing barrier / max-over-ranks here.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

TOTAL_ENVS = 16384
HORIZON = 32
MINIBATCH = 16384      # im.yaml:72 (per rank, as under Horovod)
MINI_EPOCHS = 6        # im.yaml:73
ALGO_BYTES_PER_ENV_STEP = 9396  # SURVEY.md 8(d): fused step kernel, core total incl. power term
METRIC = "env-steps/sec at 16384 humanoid envs, 1/2/4/8 H100; obs-kernel HBM GB/s"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--envs", type=int, default=TOTAL_ENVS)
    ap.add_argument("--median-frames", type=int, default=150)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the outputs of the last timed PPO iteration (a fixed sample of the experience rows "
                         "and the updated policy) to DIR/<name>.npy, float32 / float64, at most 64 MB in all")
    ap.add_argument("--workload", default="ppo", choices=["ppo", "vae", "reach"],
                    help="ppo = the headline (BASELINE configs[3], the default the driver runs); vae = configs[2] PULSE VAE distillation, "
                         "8192 envs; reach = configs[4] latent reach task (1024 envs per GPU): single-GPU records of the secondary workloads")
    return ap.parse_args()


class ClockSampler(threading.Thread):
    """Samples SM clocks / throttle reasons with nvidia-smi during the timed region."""

    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.samples, self._stop_evt = index, [], threading.Event()

    def run(self):
        while not self._stop_evt.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", str(self.index)],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.samples.append([x.strip() for x in out.split(",")])
            except Exception:
                pass
            self._stop_evt.wait(0.1)

    def stop(self):
        self._stop_evt.set()
        self.join(timeout=5)
        sm, reasons, mx = [], set(), None
        for s in self.samples:
            try:
                sm.append(float(s[0]))
                mx = float(s[1])
            except Exception:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), s[2:6]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


# --------------------------------------------------------------------------------------------------
def pick_cpu_threads(max_threads):
    """PyTorch CPU ops on [N,24,4]-sized tensors stop scaling (and can collapse) long before 128
    threads; give the CPU arm the thread count at which it runs fastest on this host."""
    best, best_rate = 1, 0.0
    for t in sorted({1, 4, 8, 16, 32, 64, max_threads}):
        if t > max_threads:
            continue
        rate, _ = cpu_port_rate(2048, 1, t, gae=True)      # chosen on the sample that is then timed
        if rate > best_rate:
            best, best_rate = t, rate
    return best


def cpu_port_rate(n_envs, n_iters, threads, gae=True):
    """Reference path on the host CPU: the oracle port of get_motion_state x2 + reward + reset + self/task
    obs + AMP obs + GAE, timed per env-step on a bounded sample."""
    import torch
    from oracle import pulse_oracle as po
    from tests.helpers import synthetic_step_inputs, synthetic_tables
    torch.set_num_threads(threads)
    tb = synthetic_tables(min(n_envs, 2048), seed=0)
    z = synthetic_step_inputs(tb, n_envs, seed=1)
    cfg = po.ImStepConfig()
    amp = torch.zeros(n_envs, 10, 196)
    T = HORIZON
    r, v, nv = (torch.randn(T, n_envs, 1) for _ in range(3))
    d = (torch.rand(T, n_envs) < 0.05).float()

    # per-step env reset of ~5 % of the envs (amp_agent.py:352 -> humanoid.py:526-609, humanoid_amp.py:468-597): the oracle's composite
    reset_ids = torch.arange(0, n_envs, 20)
    phase = torch.rand(n_envs)
    st = {"motion_ids": z["motion_ids"], "start_times": z["start_times"], "start_offset": z["start_offset"], "global_offset": z["global_offset"],
          "cycle_counter": z["cycle_counter"], "progress_buf": z["progress_buf"], "reset_buf": z["reset_buf_in"],
          "terminate_buf": z["reset_buf_in"], "root_states": z["body_state"][:, 0].clone(), "dof_pos": z["dof_pos"], "dof_vel": z["dof_vel"],
          "body_state": z["body_state"], "contact_forces": torch.zeros(n_envs, 24, 3), "amp_obs_buf": amp, "obs_buf": torch.zeros(n_envs, 934),
          "dof_force": z["dof_force"]}

    def one_env_step():
        po.reset_envs(tb, cfg, st, reset_ids, phase)
        po.humanoid_im_step(tb, cfg, z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"],
                            z["start_times"], z["start_offset"], z["global_offset"], z["cycle_counter"], z["reset_buf_in"])
        return po.amp_obs_step(amp, z["body_state"], z["dof_pos"], z["dof_vel"])

    def gae_pass():
        adv = po.discount_values(d, v, r, nv)
        return po.normalized_advantages(po.swap_and_flatten01(adv + v), po.swap_and_flatten01(v))

    # networks of im.yaml as plain fp32 torch modules (what the reference trains: mixed_precision False, im.yaml:51)
    def mlp(i, o):
        return torch.nn.Sequential(torch.nn.Linear(i, 1024), torch.nn.ReLU(), torch.nn.Linear(1024, 512), torch.nn.ReLU(), torch.nn.Linear(512, o))
    actor, critic, disc = mlp(934, 69), mlp(934, 1), mlp(1960, 1)
    params = list(actor.parameters()) + list(critic.parameters()) + list(disc.parameters())
    opt = torch.optim.Adam(params, lr=2e-5, eps=1e-8)
    obs = torch.randn(n_envs, 934)
    ampx = torch.randn(n_envs, 1960)
    logstd = torch.full((69,), -2.9)
    adv_b, ret_b = torch.randn(n_envs), torch.randn(n_envs)

    def rollout_nets():
        with torch.no_grad():
            x = torch.clamp(obs, -5, 5)
            mu = actor(x)
            critic(x)
            critic(x)                      # next-value evaluation
            disc(torch.clamp(ampx, -5, 5))
            a_ = mu + torch.exp(logstd) * torch.randn_like(mu)
            return a_, po.gaussian_neglogp(a_, mu, torch.exp(logstd).expand_as(mu), logstd.expand_as(mu))

    def update_minibatch(a_, nlp):
        x = torch.clamp(obs, -5, 5)
        out = po.ppo_total_loss(actor(x), critic(x).squeeze(1), nlp, adv_b, ret_b, a_, logstd)
        q = max(1, n_envs // 4)            # amp_minibatch_size / minibatch_size = 4096 / 16384
        ax = torch.clamp(ampx, -5, 5)
        dl = po.disc_loss(disc, ax[:q], ax[q:2 * q], ax[2 * q:3 * q], disc[4].weight, [disc[0].weight, disc[2].weight, disc[4].weight])
        opt.zero_grad(set_to_none=True)
        (out["loss"] + 5.0 * dl["disc_loss"]).backward()
        torch.nn.utils.clip_grad_norm_(params, 50.0)
        opt.step()

    one_env_step()
    t0 = time.perf_counter()
    for _ in range(n_iters):
        one_env_step()
    t_step = (time.perf_counter() - t0) / n_iters
    t_gae = t_net = t_upd = 0.0
    if gae:
        gae_pass()
        t0 = time.perf_counter()
        gae_pass()
        t_gae = time.perf_counter() - t0
        a_, nlp = rollout_nets()
        t0 = time.perf_counter()
        a_, nlp = rollout_nets()
        t_net = time.perf_counter() - t0
        update_minibatch(a_, nlp)
        t0 = time.perf_counter()
        update_minibatch(a_, nlp)
        t_upd = time.perf_counter() - t0
    # one PPO iteration over n_envs: 32 env steps (+ net forwards), GAE, 6 epochs x 32 minibatches of n_envs rows
    per_iter = HORIZON * (t_step + t_net) + t_gae + MINI_EPOCHS * HORIZON * t_upd
    return HORIZON * n_envs / per_iter, per_iter


def run_reference(a):
    """--impl reference: the reference's CPU path (oracle port), all host threads, bounded sample."""
    import torch
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = pick_cpu_threads(os.cpu_count() or 1)
    n = min(a.envs, 2048)
    vals, per = [], []
    for i in range(a.warmup + a.steps):
        rate, per_iter = cpu_port_rate(n, 2, threads)
        if i >= a.warmup:
            vals.append(rate)
            per.append(per_iter)
    value = sum(vals) / len(vals)
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": "env-steps/s", "n_gpus": a.gpus, "steps": a.steps, "warmup": a.warmup,
        "ms_per_step": 1e3 * sum(per) / len(per) * (a.envs / n), "extrapolated": True,
        "sample_seconds_measured": sum(per) / len(per) / (HORIZON * (1 + MINI_EPOCHS)) * 3,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": workload_config(a, 1, a.envs),
        "cpu_baseline": {"value": value, "unit": "env-steps/s", "cores": threads, "host_cores": os.cpu_count(), "kind": "port",
                         "sample": f"{n} envs: 2 env-steps (5% env resets + obs/reward/reset/AMP) + policy/critic/disc fwd + one PPO minibatch fwd/bwd/Adam + GAE, "
                                   f"fp32; value and ms_per_step are EXTRAPOLATED from that sample to a 32-step iteration with 6 mini-epochs of {a.envs} envs "
                                   f"(thread count chosen on the same 2048-env sample); torch {torch.__version__} CPU"},
        "e2e": {"value": value, "unit": "env-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


def workload_config(a, world, envs_total):
    mb = HORIZON * (envs_total // world) // MINIBATCH
    return {
        "workload": "HumanoidIm PPO iteration, 16384 envs total, AMASS-shaped synthetic MotionLib (one clip per env, "
                    f"lognormal lengths, median {a.median_frames} frames @30fps), horizon 32, im.yaml nets (BASELINE configs[3])",
        "envs_total": envs_total, "envs_per_gpu": envs_total // world, "horizon": HORIZON, "minibatch": MINIBATCH,
        "mini_epochs": MINI_EPOCHS, "minibatches_per_epoch_per_gpu": mb, "parallelism": f"env-shard x{world}, grad all-reduce per minibatch",
        "phases": ["32x fused env reset of the done envs, no host sync (pulse_reset_ref_state: compaction, start-time draw, MotionLib query, scatter into "
                   "root / dof / rigid-body state, AMP history back-fill) + observation of the reset envs (a13)",
                   "32x [obs normalise + actor/critic MLP fwd (wgmma) + in-kernel Gaussian sample, neglogp, value de-normalisation, PD targets, "
                   "written straight into the experience slices (K7-K9, K22)]",
                   "32x fused progress += 1 + reward + reset + next observation kernel (K1-K5)", "32x AMP observation row written into its experience slice (K6)",
                   "32x critic fwd on the next obs -> next_values * (1 - terminated)", "discriminator fwd + AMP reward over 32xN rows (K10)",
                   "GAE + returns + adv-norm (K11,K12)", "value/return normalisation (running stats)",
                   f"{MINI_EPOCHS} mini-epochs x minibatches: obs-RMS update, actor/critic fwd, PPO loss, bwd (dgrad+wgrad), "
                   "discriminator loss on 3x4096 AMP rows: BCE + logit reg + weight decay + ANALYTIC gradient penalty (K14), "
                   "NCCL gradient averaging per network chain on its own stream / communicator, overlapped with the other chains (N>1), "
                   "grad-norm clip + Adam incl. bf16 operand mirror (K13,K15,K16); per mini-epoch KL average and per-epoch RunningMeanStd sync across "
                   "ranks (N>1; common_agent.py:126-127, amp_agent.py:523-524)",
                   "AMP demo fetch (MotionLib query + AMP obs), demo / replay ring updates and per-minibatch draws"],
        "not_yet": ["physics (gym.simulate + refresh/set tensor calls): excluded on every arm",
                    "rl_games bookkeeping outside the arithmetic: episode reward / length meters, tensorboard / wandb logging, checkpoint writes",
                    "AMP replay-buffer insertion uses a fixed-size random subset (amp_replay_keep_prob) instead of a Bernoulli mask"],
        "physics": "excluded (Isaac Gym not installable; simulator state tensors are synthetic, resident in HBM)",
        "l2": "256 MiB L2 flush write before every timed iteration; per-iteration working set (tables 3.9 GB + 6 GB rollout buffers at N=1) exceeds L2",
    }


# per env-step ALGORITHMIC MLP FLOPs inside the timed region (2 x MAC), im.yaml nets (K = 934 / 1960: the zero padding to 960 the
# operands carry is not counted)
def mlp_flops_per_env_step():
    a = 934 * 1024 + 1024 * 512 + 512 * 69     # actor fwd MACs
    c = 934 * 1024 + 1024 * 512 + 512 * 1      # critic fwd MACs
    d = 1960 * 1024 + 1024 * 512 + 512 * 1     # disc fwd MACs
    rollout = a + 2 * c + d                    # actor + critic (values) + critic (next values) + disc reward
    # update: fwd + wgrad for every layer, dgrad for all but the first layer of each net
    dgrad_a = 1024 * 512 + 512 * 69
    dgrad_c = 1024 * 512 + 512 * 1
    # discriminator update: 3 x 4096 rows per 16384-row minibatch (0.75 rows/row): fwd + wgrad + dgrad(2 upper layers),
    # plus on the 4096 demo rows the analytic gradient penalty: 2 input-gradient GEMMs + 2 wgrad + 2 NT GEMMs
    dg = 1024 * 512 + 512 * 1
    gp = (512 * 1024 + 1024 * 1960) + (1024 * 1960 + 512 * 1024) + (1960 * 1024 + 1024 * 512)
    disc_upd = MINI_EPOCHS * (0.75 * (2 * d + dg) + 0.25 * gp)
    update = MINI_EPOCHS * (2 * (a + c) + dgrad_a + dgrad_c) + disc_upd
    return 2.0 * (rollout + update)


SECONDARY = {
    "vae": ("env-steps/sec, PULSE VAE distillation (encoder + prior + decoder MLP), 8192 humanoid envs, 1 H100 (BASELINE configs[2])", 8192),
    "reach": ("env-steps/sec, latent-space reach task with the frozen PULSE decoder, 1024 envs per H100 (BASELINE configs[4]: 8192 envs on 8 GPUs)", 1024),
}


def cpu_secondary_rate(workload, threads):
    """CPU port (oracle) of one minibatch update + one env step of a secondary workload on a bounded sample, extrapolated to an iteration."""
    import torch
    from oracle import pulse_oracle as po
    from tests.helpers import VAE_FULL, synthetic_step_inputs, synthetic_tables, vae_full_fixture, vae_param_list
    torch.set_num_threads(threads)
    n = 512
    tb = synthetic_tables(n, seed=0)
    z = synthetic_step_inputs(tb, n, seed=1)
    cfg = po.ImStepConfig()
    t0 = time.perf_counter()
    po.humanoid_im_step(tb, cfg, z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"], z["start_times"], z["start_offset"],
                        z["global_offset"], z["cycle_counter"], z["reset_buf_in"])
    t_step = (time.perf_counter() - t0) / n                         # seconds per env-step of the obs / reward / reset path
    if workload == "vae":
        sd, batch, _ = vae_full_fixture()
        nets = po.VaeNets.from_state_dict(sd, VAE_FULL["S"])
        params = [p.requires_grad_(True) for p in vae_param_list(nets).values()]
        opt = torch.optim.Adam(params, lr=5e-4)
        rows = batch["obs"].shape[0]

        def upd():
            opt.zero_grad(set_to_none=True)
            r = po.vae_kin_loss(nets, batch["obs"], batch["noise"], batch["gt_action"], batch["progress"], VAE_FULL["T"])
            r["kin_loss"].backward()
            torch.nn.utils.clip_grad_norm_(params, 50.0)
            opt.step()
        upd()
        t0 = time.perf_counter()
        upd()
        t_upd = (time.perf_counter() - t0) / rows                    # seconds per row of one _optimize_kin minibatch
        with torch.no_grad():
            t0 = time.perf_counter()
            po.vae_eval_actor(nets, batch["obs"], batch["noise"])
            t_fwd = (time.perf_counter() - t0) / rows
        per_env_step = t_step + 2 * t_fwd + MINI_EPOCHS * t_upd      # rollout: student forward + teacher of comparable size
        return 1.0 / per_env_step, f"{rows}-row _optimize_kin minibatch (im_z_fit.yaml nets, fwd + autograd bwd + Adam) + encoder/decoder forward + {n}-env step path"
    lin = lambda i, o: torch.nn.Linear(i, o)
    mk = lambda i, o: torch.nn.Sequential(lin(i, 2048), torch.nn.SiLU(), lin(2048, 1024), torch.nn.SiLU(), lin(1024, 512), torch.nn.SiLU(), lin(512, o))
    actor, critic = mk(361, 32), mk(361, 1)
    params = list(actor.parameters()) + list(critic.parameters())
    opt = torch.optim.Adam(params, lr=2e-5)
    rows = 2048
    obs, act = torch.randn(rows, 361), torch.randn(rows, 32)
    logstd = torch.full((32,), -2.9)
    adv, ret, nlp = torch.randn(rows), torch.randn(rows), torch.randn(rows) + 20

    def upd():
        opt.zero_grad(set_to_none=True)
        out = po.ppo_total_loss(actor(obs), critic(obs).squeeze(1), nlp, adv, ret, act, logstd)
        out["loss"].backward()
        torch.nn.utils.clip_grad_norm_(params, 50.0)
        opt.step()
    upd()
    t0 = time.perf_counter()
    upd()
    t_upd = (time.perf_counter() - t0) / rows
    with torch.no_grad():
        t0 = time.perf_counter()
        actor(obs); critic(obs); critic(obs)
        t_fwd = (time.perf_counter() - t0) / rows
    per_env_step = 0.4 * t_step + 3 * t_fwd + MINI_EPOCHS * t_upd   # reach obs is the 358-float self observation part of the step path
    return 1.0 / per_env_step, f"{rows}-row PPO minibatch of the pulse_z_task.yaml policy (fwd + autograd bwd + Adam) + policy/critic/decoder-sized forwards + step path"


def run_secondary(a):
    import torch
    metric, envs = SECONDARY[a.workload]
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return                                                        # single-GPU records: the other ranks of a torchrun launch exit without work
    if a.impl == "reference":
        threads = min(os.cpu_count() or 1, 32)
        vals = []
        for i in range(a.warmup + a.steps):
            rate, sample = cpu_secondary_rate(a.workload, threads)
            if i >= a.warmup:
                vals.append(rate)
        value = sum(vals) / len(vals)
        line = {"impl": "reference", "metric": metric, "value": value, "unit": "env-steps/s", "n_gpus": a.gpus, "steps": a.steps, "warmup": a.warmup,
                "ms_per_step": 1e3 * HORIZON * envs / value, "extrapolated": True, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "f32", "data": "synthetic", "config": {"workload": metric, "envs": envs},
                "cpu_baseline": {"value": value, "unit": "env-steps/s", "cores": threads, "host_cores": os.cpu_count(), "kind": "port", "sample": sample},
                "e2e": {"value": value, "unit": "env-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line), flush=True)
        return
    from tools import bench_pulse
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    ns = argparse.Namespace(envs=envs if a.envs == TOTAL_ENVS else a.envs, steps=a.steps, warmup=a.warmup)
    sampler = ClockSampler(0)
    sampler.start()
    out = bench_pulse.bench_vae(ns, dev) if a.workload == "vae" else bench_pulse.bench_reach(ns, dev)
    clocks = sampler.stop()
    line = {"metric": metric, "value": out["value"], "unit": "env-steps/s", "n_gpus": 1, "steps": a.steps, "warmup": a.warmup,
            "ms_per_step": out["ms_per_iteration"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16 GEMM operands, fp32 accumulate / master weights / observations", "data": "synthetic",
            "config": {"workload": out["workload"], "envs": ns.envs, "horizon": HORIZON, "minibatch": MINIBATCH, "mini_epochs": MINI_EPOCHS,
                       "phases": out["phases"], "not_yet": out.get("not_run", []) + ["physics (excluded on every arm)"], "l2": out["l2"]},
            "e2e": out["e2e"], "gpu_launches": out["gpu_launches"], "cuda_graphs": out["cuda_graphs"], "clocks": clocks,
            "roofline": dict(out["roofline_update"], kernel="gemm_bf16_kernel family (update phase)", traffic=None),
            "phases_ms": {"rollout": out["rollout_ms"], "update": out["update_ms"]}, "mlp_mflop_per_env_step": out["mflop_per_env_step"]}
    if not a.no_cpu_baseline:
        threads = min(os.cpu_count() or 1, 32)
        rate, sample = cpu_secondary_rate(a.workload, threads)
        line["cpu_baseline"] = {"value": rate, "unit": "env-steps/s", "cores": threads, "host_cores": os.cpu_count(), "kind": "port", "extrapolated": True,
                                "sample": sample}
    print(json.dumps(line), flush=True)


def dump_outputs(out_dir, ps, policy, rows=2048, amp_rows=1024, limit=64 << 20):
    """What the last timed PPO iteration handed its caller: the experience of the rollout (a fixed sample of `rows` of the n x 32
    rows; `amp_rows` of the 1960-wide AMP rows) and the policy after the update (weights, log-std, normaliser statistics)."""
    import numpy as np
    import torch
    torch.cuda.synchronize()
    n_rows = ps.n * ps.T
    idx = torch.from_numpy(np.sort(np.random.RandomState(0).choice(n_rows, size=min(rows, n_rows), replace=False))).to(ps.dev)
    arrays = {}
    for name in ("obses", "actions", "mus", "neglogp", "values", "next_values", "rewards", "dones", "adv", "ret", "amp_obs"):
        t = getattr(ps, name).reshape(n_rows, -1)
        arrays["rollout." + name] = t.index_select(0, idx[:amp_rows] if name == "amp_obs" else idx)
    arrays.update(policy.state_dict())
    host = {}
    for name, t in arrays.items():
        x = t.detach().cpu().numpy()
        host[name] = x.astype(np.float64 if x.dtype == np.float64 else np.float32)
    total = sum(x.nbytes for x in host.values())
    if total > limit:                          # checked before anything is written: no partial DIR
        raise SystemExit(f"--dump-outputs: {total >> 20} MB exceeds {limit >> 20} MB")
    os.makedirs(out_dir, exist_ok=True)
    for name, x in host.items():
        np.save(os.path.join(out_dir, name + ".npy"), x)


def main():
    a = parse()
    if a.workload != "ppo":
        return run_secondary(a)
    if a.impl == "reference":
        return run_reference(a)
    import torch
    import torch.distributed as dist
    from pulse_b200 import _lib
    from pulse_b200.humanoid_im import HumanoidImCompute
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.nets import pad_k
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.rollout import discount_values
    from pulse_b200.vae import pd_targets
    from tools.synth import device_step_inputs, device_tables

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == a.gpus, f"--gpus {a.gpus} but WORLD_SIZE={world} (launch with torch.distributed.run)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    # every draw without an explicit generator (AMP demo sampling, replay ring, minibatch indices) comes from these seeds: the same
    # arguments give the same inputs on every run
    torch.manual_seed(0)
    if world > 1:
        # NCCL prints its version banner on STDOUT when the communicator is created (NCCL_DEBUG >= VERSION in the environment);
        # stdout must carry exactly one JSON line, so fd 1 points at stderr until the communicator exists.
        sys.stdout.flush()
        saved_fd = os.dup(1)
        os.dup2(2, 1)
        try:
            dist.init_process_group("nccl", device_id=dev)
            warm = torch.zeros(1, device=dev)
            dist.all_reduce(warm)
            torch.cuda.synchronize()
        finally:
            sys.stdout.flush()
            os.dup2(saved_fd, 1)
            os.close(saved_fd)
    n = a.envs // world
    lib = _lib.load()
    T = HORIZON
    assert (T * n) % MINIBATCH == 0, "rollout batch must be a multiple of the minibatch"
    num_mb = T * n // MINIBATCH

    # ---- synthetic inputs, resident in HBM (shard: envs [rank*n, (rank+1)*n), one clip per env) ----
    tabs = device_tables(n, dev, seed=100 + rank, median_frames=a.median_frames)
    ml = MotionLibB200.from_tables(tabs)
    del tabs
    z = device_step_inputs(ml, n, seed=200 + rank)
    comp = HumanoidImCompute(ml)
    os.environ.setdefault("PULSE_PEER_TIMEOUT_MS", "120000")  # ranks of a bench run stay in lock step: a peer missing for 2 min is a failure
    policy = PPOPolicy(device=dev, seed=0, with_disc=True)   # replicated: same seed on every rank (Horovod broadcast equivalent)
    disc = policy.disc
    AMP_MB = 4096                                        # amp_minibatch_size (im.yaml:81)
    REPLAY = 200000                                      # amp_replay_buffer_size / amp_obs_demo_buffer_size (im.yaml:77-78)
    replay_buf = torch.randn(REPLAY, 1960, device=dev)   # AMP replay ring (amp_agent.py:1043-1057), pre-filled
    demo_buf = comp.fetch_amp_obs_demo(512).repeat((REPLAY + 511) // 512, 1)[:REPLAY].contiguous()   # demo ring (_init_amp_demo_buf)
    replay_mb = torch.zeros(num_mb, AMP_MB, 1960, device=dev)
    demo_mb = torch.zeros(num_mb, AMP_MB, 1960, device=dev)
    ring_pos = [0]

    # ---- the rollout driver: AMPAgent.play_steps on the device (pulse_b200/rollout.py), experience buffers ENV-MAJOR ----------------
    from pulse_b200.rollout import PlayStepsB200
    root_states = torch.zeros(n, 1, 13, device=dev)        # _humanoid_root_states view of the actor root tensor (humanoid.py:197-200)
    root_states[:, 0] = z["body_state"][:, 0]
    contact = torch.zeros(n, z["body_state"].shape[1], 3, device=dev)
    sim = dict(body_state=z["body_state"], root_states=root_states[:, 0], dof_pos=z["dof_pos"], dof_vel=z["dof_vel"], dof_force=z["dof_force"],
               progress_buf=z["progress_buf"], motion_ids=z["motion_ids"], motion_start_times=z["motion_start_times"],
               motion_start_offset=z["motion_start_offset"], global_offset=z["global_offset"], cycle_counter=z["cycle_counter"],
               contact_forces=contact, actor_ids=torch.arange(n, dtype=torch.int32, device=dev))
    pd_offset, pd_scale = torch.zeros(69, device=dev), torch.full((69,), 1.2, device=dev)   # _build_pd_action_offset_scale (humanoid.py:492-543)
    use_graphs = os.environ.get("PULSE_NO_GRAPHS", "0") != "1"
    single_graph = os.environ.get("PULSE_ROLLOUT_GRAPH", "1") != "0"
    ps = PlayStepsB200(comp, policy, sim, horizon=T, pd_offset=pd_offset, pd_scale=pd_scale, use_graphs=use_graphs, single_graph=single_graph,
                       reset_seed=1000 + rank)
    ps.first_observation()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    # pinned host mirrors for the end-to-end arm: the simulator state is re-uploaded before every env step, rewards / resets read back
    h_body = z["body_state"].cpu().pin_memory()
    h_dof = z["dof_state"].cpu().pin_memory()
    h_force = z["dof_force"].cpu().pin_memory()
    h_rew = torch.empty(n, dtype=torch.float32).pin_memory()
    h_reset = torch.empty(n, dtype=torch.float32).pin_memory()
    h_term = torch.empty(n, dtype=torch.long).pin_memory()
    h2d = h_body.numel() * 4 + h_dof.numel() * 4 + h_force.numel() * 4
    d2h = n * (4 + 4 + 8)

    def upload(t):
        z["body_state"].copy_(h_body, non_blocking=True)
        z["dof_state"].copy_(h_dof, non_blocking=True)
        z["dof_force"].copy_(h_force, non_blocking=True)

    def download(t):
        h_rew.copy_(ps.rewards[t], non_blocking=True)
        h_reset.copy_(ps.dones[t], non_blocking=True)
        h_term.copy_(ps.terminate_buf, non_blocking=True)

    update_events = []
    done_frac = torch.zeros(1, device=dev)
    obs_f, act_f, mu_f, nlp_f = ps.obses.view(T * n, 934), ps.actions.view(T * n, 69), ps.mus.view(T * n, 69), ps.neglogp.view(T * n)
    amp_f = ps.amp_obs.view(n * T, 1960)

    def post_rollout():
        # AMP demo / replay bookkeeping of train_epoch (amp_agent.py:476-483, :998-1001, :1043-1057): new demo samples into the
        # demo ring, this rollout's AMP observations into the replay ring, one random draw per minibatch from each
        new_demo = comp.fetch_amp_obs_demo(512)
        p0 = ring_pos[0] % (REPLAY - 512)
        demo_buf[p0:p0 + 512].copy_(new_demo)
        idx = torch.randint(0, REPLAY, (num_mb * AMP_MB,), device=dev)
        torch.index_select(replay_buf, 0, idx, out=replay_mb.view(-1, 1960))
        idx2 = torch.randint(0, REPLAY, (num_mb * AMP_MB,), device=dev)
        torch.index_select(demo_buf, 0, idx2, out=demo_mb.view(-1, 1960))
        keep = torch.randint(0, n * T, (2048,), device=dev)                       # amp_replay_keep_prob 0.01 of the batch
        replay_buf[p0:p0 + 2048].copy_(amp_f[keep])
        ps.finish()            # disc rewards, reward mix, GAE, advantage + value / return normalisation (rollout.py)
        done_frac.add_(ps.dones.mean())

    def mb_inputs(i):
        r0 = i * MINIBATCH
        return obs_f[r0:r0 + MINIBATCH], (amp_f[r0:r0 + AMP_MB], replay_mb[i], demo_mb[i])   # amp_obs[0:amp_minibatch_size] (amp_agent.py:621-628)

    # The weight-independent head of a minibatch (observation / AMP normalisation with their running-statistics updates) is prepared
    # one minibatch ahead on a side stream, in the reference's order, into the other operand slot (PULSE_PREFETCH=0: inline).
    prefetching = os.environ.get("PULSE_PREFETCH", "1") != "0" and num_mb % 2 == 0

    def prepare_first():
        policy.prepare_inputs(*mb_inputs(0), slot=0)

    def update_mb(i, last=False):
        r0, r1 = i * MINIBATCH, (i + 1) * MINIBATCH
        obs_i, amp_i = mb_inputs(i)
        kw = {}
        if prefetching:
            kw = dict(slot=i & 1, prepared=True, prefetch=None if last else mb_inputs((i + 1) % num_mb))
        policy.train_minibatch(obs_i, act_f[r0:r1], nlp_f[r0:r1], ps.adv[r0:r1], ps.ret[r0:r1], old_mu=mu_f[r0:r1], world_size=world,
                               amp=amp_i, **kw)

    # ---- CUDA graphs: every launch sequence with fixed buffers is captured once and replayed -----------------
    graphs = {}
    pool = torch.cuda.graph_pool_handle() if use_graphs else None   # replays are sequential: one shared private pool

    def run(key, fn, *args):
        if not use_graphs:
            return fn(*args)
        g = graphs.get(key)
        if g is None:                                   # first use: eager (lazy workspaces, one-time attribute calls)
            graphs[key] = False
            return fn(*args)
        if g is False:                                  # second use: capture (records only), then replay = this use's one execution
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=pool):
                fn(*args)
            graphs[key] = g
        g.replay()

    step_ms = []

    phase_events = []

    def iteration(e2e, record):
        ps.host_io = (upload, download) if e2e else None
        if record:
            r0, r1, us, ue = (torch.cuda.Event(enable_timing=True) for _ in range(4))
            r0.record()
        ps.play_steps()
        if record:
            r1.record()
        run(("post_rollout",), post_rollout)
        if record:
            us.record()
            phase_events.append((r0, r1, us))
        if prefetching:
            run(("prepare_first",), prepare_first)
        for ep in range(MINI_EPOCHS):
            policy.reset_stats()                           # loss / KL statistics accumulate over the mini-epoch's minibatches
            for i in range(num_mb):
                last = prefetching and ep == MINI_EPOCHS - 1 and i == num_mb - 1      # nothing left to prepare
                run(("upd", i, last), update_mb, i, last)
            if world > 1:                                  # av_kls = hvd.average_value(av_kls) per mini-epoch (amp_agent.py:523-524)
                dist.all_reduce(policy.stats, op=dist.ReduceOp.AVG)
        if world > 1:                                      # hvd.sync_stats once per epoch (common_agent.py:126-127)
            policy.sync_stats(world)
        if record:
            ue.record()
            update_events.append((us, ue))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(e2e, steps, record):
        for _ in range(a.warmup):
            flush.fill_(1)
            iteration(e2e, False)
        barrier()
        launches0 = lib.pulse_launch_count()
        total_ms = 0.0
        for _ in range(steps):
            flush.fill_(1)  # L2 flush, outside the timed span
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            barrier()
            s.record()
            iteration(e2e, record)
            e.record()
            barrier()
            if record:
                step_ms.extend(ps.step_kernel_ms())     # graph-safe events around every fused step kernel of this iteration
            ms = torch.tensor([s.elapsed_time(e)], device=dev)
            if world > 1:
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            total_ms += float(ms.item())
        return total_ms / steps, (lib.pulse_launch_count() - launches0) // steps

    # count our kernels per iteration once, eagerly (graph replays do not pass through the library's counter)
    use_graphs, saved = False, use_graphs
    ps.use_graphs = False
    iteration(False, False)
    l0 = lib.pulse_launch_count()
    iteration(False, False)
    launches_eager = lib.pulse_launch_count() - l0
    use_graphs = ps.use_graphs = saved
    done_frac.zero_()
    iters_counted = [0]

    sampler = ClockSampler(local)
    sampler.start()
    ms_dev, launches = timed(False, a.steps, True)
    clocks = sampler.stop()
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, ps, policy)
    ms_e2e, _ = timed(True, max(2, a.steps // 2), False)

    torch.cuda.synchronize()
    k_ms = sorted(step_ms)
    k_avg = sum(k_ms) / len(k_ms)
    u_ms = sum(s.elapsed_time(e) for s, e in update_events) / len(update_events)
    rollout_ms = sum(a0.elapsed_time(a1) for a0, a1, _ in phase_events) / len(phase_events)
    post_ms = sum(a1.elapsed_time(a2) for _, a1, a2 in phase_events) / len(phase_events)
    n_iters_total = 2 * a.warmup + a.steps + max(2, a.steps // 2)          # iterations since done_frac was cleared
    resets_per_step = float(done_frac.item()) / n_iters_total
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    # fallbacks: NVIDIA's H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense BF16 at up to 700 W), not reached figures
    peak = float(peaks.get("hbm_gbs", 3350.0))
    peak_tf = float(peaks.get("bf16_tflops_sustained", 989.0))
    achieved = ALGO_BYTES_PER_ENV_STEP * n / (k_avg * 1e-3) / 1e9
    env_steps = T * a.envs
    _d = 1960 * 1024 + 1024 * 512 + 512
    _gp = 3 * (512 * 1024 + 1024 * 1960)
    upd_flops = 2.0 * MINI_EPOCHS * (2 * (934 * 1024 + 1024 * 512 + 512 * 69 + 934 * 1024 + 1024 * 512 + 512)
                                     + 2 * 1024 * 512 + 512 * 69 + 512
                                     + 0.75 * (2 * _d + 1024 * 512 + 512) + 0.25 * _gp) * T * n
    if rank == 0:
        line = {
            "metric": METRIC, "value": env_steps / (ms_dev * 1e-3), "unit": "env-steps/s", "n_gpus": world, "steps": a.steps,
            "warmup": a.warmup, "ms_per_step": ms_dev, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "bf16 GEMM operands, fp32 accumulate / master weights / observations", "data": "synthetic",
            "config": workload_config(a, world, a.envs),
            "e2e": {"value": env_steps / (ms_e2e * 1e-3), "unit": "env-steps/s", "h2d_bytes_per_step": T * h2d * world,
                    "d2h_bytes_per_step": T * d2h * world, "ms_per_step": ms_e2e},
            "gpu_launches": int(launches_eager), "cuda_graphs": bool(use_graphs), "rollout_single_graph": bool(use_graphs and single_graph),
            "clocks": clocks,
            "phases_ms": {"rollout_32_steps": rollout_ms, "post_rollout": post_ms, "update": u_ms,
                          "note": "device-resident arm, this rank; rollout = resets + policy + fused step + AMP + next values per step"},
            "resets_per_env_step": resets_per_step,
            "gemm_switches": {"pdl": os.environ.get("PULSE_GEMM_PDL", "1") != "0",
                              "grouped_launches": os.environ.get("PULSE_GROUPED", "0") == "1"},
            "update_input_prefetch": bool(prefetching),
            "optimizer_step": ("one peer-memory kernel per rank: reduce-scatter over NVLink + norm clip + sharded Adam + push of masters / bf16 operands"
                               + (" (multimem)" if policy.flat.peer and policy.flat.peer["multicast"] else "")) if (world > 1 and policy.flat.peer)
                              else ("ncclAllReduce(AVG) + sum_squares + adam" if world > 1 else "sum_squares + adam (single GPU)"),
            "roofline": {"kernel": "im_step_kernel", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                         "frac": achieved / peak, "traffic": None,
                         "algorithmic_bytes_per_launch": ALGO_BYTES_PER_ENV_STEP * n,
                         "peak_source": "MEASURED_PEAKS.json hbm_gbs (of measured)" if peaks else "H100 SXM data sheet 3350",
                         "algorithmic_bytes_per_env_step": ALGO_BYTES_PER_ENV_STEP, "avg_launch_ms": k_avg, "launches_timed": len(k_ms)},
            "roofline_update": {"kernels": "PPO update phase (wgmma GEMMs + loss/Adam/reduction kernels), per rank", "bound": "tensor",
                                "achieved": upd_flops / (u_ms * 1e-3) / 1e12, "peak": peak_tf, "unit": "TFLOP/s",
                                "frac": upd_flops / (u_ms * 1e-3) / 1e12 / peak_tf, "update_ms": u_ms,
                                "peak_source": "MEASURED_PEAKS.json bf16_tflops_sustained (of measured)" if peaks else "H100 SXM data sheet 989 (dense bf16)",
                                "note": "algorithmic GEMM FLOPs of the update / whole update-phase time (non-GEMM kernels included)"},
            "mlp_mflop_per_env_step": mlp_flops_per_env_step() / 1e6,
        }
        if not a.no_cpu_baseline:
            threads = pick_cpu_threads(os.cpu_count() or 1)
            rate, per_iter = cpu_port_rate(2048, 2, threads)
            line["cpu_baseline"] = {"value": rate, "unit": "env-steps/s", "cores": threads, "host_cores": os.cpu_count(), "kind": "port",
                                    "extrapolated": True,
                                    "sample": "2048 envs: 2 env-steps (5% env resets + obs/reward/reset/AMP) + policy fwd + one PPO minibatch fwd/bwd + GAE "
                                              "(oracle port of the reference PyTorch path, fp32), extrapolated to a 32-step iteration with 6 mini-epochs"}
        print(json.dumps(line), flush=True)
    if world > 1:
        # Leave without tearing the communicator down: destroy_process_group() was measured to hang at N=2 while CUDA graphs
        # holding captured NCCL kernels are alive.  Everything is done and printed; a barrier keeps the ranks together, then
        # every rank exits 0 directly.
        graphs.clear()
        ps._graphs.clear()
        dist.barrier()
        torch.cuda.synchronize()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)


if __name__ == "__main__":
    main()
