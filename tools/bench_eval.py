#!/usr/bin/env python
"""The evaluation pass on the device (`EvalStepsB200`) for the three `im_amp` policies: HumanoidIm (PHC, im.yaml: 934 -> 69, 1024-512
ReLU), the VR controller task (pulse_z_vr.yaml: head and hands tracked, latent policy 2048-1536-1024-1024-512-512 SiLU, frozen prior +
decoder) and, with `--policies distill`, the PULSE student of HumanoidImDistillGetup (im_z_fit.yaml / env_im_vae.yaml: encoder 934 ->
1536-1024-512-160 -> 2x32, decoder 390 -> 3096-2048-1024 -> 69, SiLU, z = the posterior mean), at --envs envs (the student: at each of
--distill-envs, by default 16384 and env_im_vae.yaml's 3072) over --clips synthetic clips (tools/synth.py, lognormal lengths at 30 fps),
no physics.

Per policy one JSON line with the card name, power limit and clocks read in the same call, and per arm
  graph   the pass as shipped: `poll_every` steps per CUDA graph, one 4-byte poll per graph
  eager   the same calls with use_graphs=False
the time of a full pass (wall clock, every chunk: load, reset, steps, read-back, the reset into training), the evaluation steps/s
(env-steps of the pass over that time) and the per-chunk host time of the chunk load (`load_motions` + the step compute) and of the
read-back of the chunk's sums.  The arms alternate pass by pass.  The student's lines add the algorithmic GEMM work of one evaluation
step from the layer shapes (multiply-accumulates per env, FLOPs = 2 MAC over the envs), the GEMM FLOP rate that implies over the pass,
and the device time of the student's action alone (normalise, encoder, Z_MEAN, decoder, PD targets; CUDA graph, CUDA events) with its
share of the graph pass.

Then one JSON line with, for comparison, the reference's per-step path at the same env count on the same frames: the MotionLib query
of body_pos_gt plus `.cpu()` copies of both position arrays every step (humanoid_im.py:662-673), and `compute_metrics_lite` over the
chunk's sequences at the end (oracle/eval_oracle.py's restatement, numpy on the host).
Needs a CUDA device: there is no fallback.

  python tools/bench_eval.py [--envs 16384] [--clips 16384] [--passes 3] [--ref-steps 64] [--policies im imz distill]
                             [--distill-envs 16384 3072]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VR = (13, 18, 23)
TABLE_KEYS = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa")


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


class DeviceDataset:
    """MotionDatasetB200's eval-side interface over device-resident synthetic tables: `load_motions` cuts the chunk's clips."""

    def __init__(self, num_unique, dev, median_frames):
        from pulse_b200.motion_dataset import MotionDatasetB200
        from tools.synth import device_tables
        self.t = device_tables(num_unique, dev, seed=7, median_frames=median_frames, max_frames=600)
        self.ds = MotionDatasetB200({f"clip_{i:05d}": {} for i in range(num_unique)}, list(range(-1, 23)), np.zeros((24, 3)), device=dev)
        self.dev, self.load_s = dev, []

    def __getattr__(self, name):
        return getattr(self.ds, name)

    def load_motions(self, n, random_sample=True, start_idx=0, max_len=-1, eval_mode=False):
        from pulse_b200.motion_lib import MotionLibB200
        t0 = time.perf_counter()
        ids = self.ds.select(n, random_sample=False, start_idx=start_idx).to(self.dev)
        nf, st = self.t["num_frames"][ids], self.t["length_starts"][ids]
        clip = torch.repeat_interleave(torch.arange(n, device=self.dev), nf)
        rows = st[clip] + (torch.arange(clip.shape[0], device=self.dev) - (torch.cumsum(nf, 0) - nf)[clip])
        tb = {k: self.t[k][rows] for k in TABLE_KEYS}
        tb.update(lengths=self.t["lengths"][ids], num_frames=nf, dt=self.t["dt"][ids], length_starts=torch.cumsum(nf, 0) - nf)
        lib = MotionLibB200.from_tables(tb, device=self.dev)
        torch.cuda.synchronize()
        self.load_s.append(time.perf_counter() - t0)
        return lib


def make_driver(kind, n, dev):
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ppo import PPOPolicy
    from tools.synth import device_step_inputs, device_tables
    ml = MotionLibB200.from_tables(device_tables(min(n, 2048), dev, seed=100, median_frames=150))
    z = device_step_inputs(ml, n, seed=200, bodies_per_env=26, dofs_per_env=72)
    root = torch.zeros(n, 2, 13, device=dev)
    root[:, 0] = z["body_state"][:, 0]
    sim = dict(body_state=z["body_state"], root_states=root[:, 0], dof_pos=z["dof_pos"], dof_vel=z["dof_vel"], progress_buf=z["progress_buf"],
               motion_ids=z["motion_ids"].clone(), motion_start_times=z["motion_start_times"], motion_start_offset=z["motion_start_offset"],
               global_offset=z["global_offset"], dof_force=z["dof_force"], cycle_counter=z["cycle_counter"],
               contact_forces=torch.zeros(n, 26, 3, device=dev), actor_ids=torch.arange(n, dtype=torch.int32, device=dev) * 2)
    if kind == "im":
        from pulse_b200.rollout import PlayStepsB200
        pol = PPOPolicy(obs_size=934, num_actions=69, units=(1024, 512), act="relu", device=dev, seed=0)
        d = PlayStepsB200(HumanoidImCompute(ml), pol, sim, horizon=32, time_steps=False)
    elif kind == "distill":
        from pulse_b200.distill import DistillStepsB200
        from pulse_b200.vae import PulseVAE, TeacherPNN
        g = torch.Generator(device=dev).manual_seed(300)
        fall_dof = torch.randn(n, 69, 2, device=dev, generator=g)
        getup = dict(recovery_counter=torch.zeros(n, dtype=torch.int32, device=dev), available_fall_states=torch.zeros(n, dtype=torch.long, device=dev),
                     fall_id_assignments=torch.zeros(n, dtype=torch.long, device=dev), fall_root_states=torch.randn(n, 13, device=dev, generator=g),
                     fall_dof_pos=fall_dof[..., 0], fall_dof_vel=fall_dof[..., 1], recovery_prob=0.5, fall_prob=0.3, recovery_steps=60)
        d = DistillStepsB200(HumanoidImCompute(ml), PulseVAE(device=dev, with_critic=False), TeacherPNN(device=dev), sim, getup, horizon=32)
    else:
        from pulse_b200.imz_rollout import ImZStepsB200
        from pulse_b200.vae import PulseVAE
        comp = HumanoidImCompute(ml, ImConfig(reset_body_ids=VR, track_body_ids=VR))
        pol = PPOPolicy(obs_size=comp.obs_size, num_actions=32, units=(2048, 1536, 1024, 1024, 512, 512), act="silu", logstd=-1.5, device=dev)
        d = ImZStepsB200(comp, pol, PulseVAE(device=dev, with_critic=False), sim, horizon=32)
    d.first_observation()
    return d


def student_macs(vae) -> int:
    """Multiply-accumulates of one student action per env: the encoder and decoder GEMMs at their unpadded layer shapes."""
    return sum(l.K * l.N for net in (vae.enc, vae.dec) for l in net.layers)


def student_step_ms(d, reps: int = 50, per_graph: int = 8) -> float:
    """Device time of the student's part of one evaluation step on its own: `eval_actor(use_mean=True)` + `pd_targets` on the driver's
    observation rows, `per_graph` of them in one CUDA graph, timed with events over `reps` replays."""
    from pulse_b200.vae import pd_targets
    pd_tar = torch.zeros(d.n, d.vae.A, device=d.dev)

    def act():
        for _ in range(per_graph):
            pd_targets(d.vae.eval_actor(d.obs_carry, use_mean=True)["mus"], d.pd[0], d.pd[1], out=pd_tar, freeze=d.pd_freeze)
    act()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        act()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps * per_graph)


def timed_pass(d, ds, use_graphs):
    from pulse_b200.evaluation import EvalMetricsB200, EvalStepsB200
    ev = EvalStepsB200(d, use_graphs=use_graphs)
    reads = []
    read = ev.metrics.read

    def timed_read():
        t0 = time.perf_counter()
        r = read()
        reads.append(time.perf_counter() - t0)
        return r
    ev.metrics.read = timed_read
    assert isinstance(ev.metrics, EvalMetricsB200)
    ds.load_s = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = ev.run(ds)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out, list(ds.load_s), reads


def reference_path(d, ds, steps):
    """Per step: MotionLib query of body_pos_gt + `.cpu()` of both position arrays; compute_metrics_lite over the sequences at the end."""
    from oracle.eval_oracle import compute_metrics_lite
    n = d.n
    lib = ds.load_motions(n, random_sample=False, start_idx=0, eval_mode=True)
    ids = torch.arange(n, device=d.dev)
    body = d.sim["body_state"]
    pred, gt = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(steps):
        times = torch.full((n,), (s + 1) * (1.0 / 30.0), device=d.dev)
        res = lib.get_motion_state(ids, times, offset=torch.zeros(n, 3, device=d.dev))
        pred.append(body[:, :24, 0:3].cpu().numpy())
        gt.append(res["rg_pos"].cpu().numpy())
    t1 = time.perf_counter()
    P, G = np.stack(pred), np.stack(gt)
    compute_metrics_lite([P[:, e] for e in range(n)], [G[:, e] for e in range(n)])
    t2 = time.perf_counter()
    return t1 - t0, t2 - t1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--clips", type=int, default=16384)
    ap.add_argument("--median-frames", type=int, default=90)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--ref-steps", type=int, default=64)
    ap.add_argument("--policies", nargs="+", default=["im", "imz"], choices=["im", "imz", "distill"])
    ap.add_argument("--distill-envs", nargs="+", type=int, default=[16384, 3072])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    dev = "cuda:0"
    info = gpu_info()
    ds = DeviceDataset(args.clips, dev, args.median_frames)
    runs = [(kind, n) for kind in args.policies for n in (args.distill_envs if kind == "distill" else [args.envs])]
    for i, (kind, n) in enumerate(runs):
        d = make_driver(kind, n, dev)
        timed_pass(d, ds, False)                                      # warm-up: module loads, lazily allocated workspaces
        res = {a: {"pass_s": [], "steps": 0, "load_s": [], "read_s": []} for a in ("graph", "eager")}
        for _ in range(args.passes):
            for a in ("graph", "eager"):
                dt, out, loads, reads = timed_pass(d, ds, a == "graph")
                r = res[a]
                r["pass_s"].append(dt)
                r["steps"] = out["steps"]
                r["chunks"] = out["chunks"]
                r["load_s"] += loads
                r["read_s"] += reads
        name = {"im": "HumanoidIm, 934 -> 69, 1024-512 ReLU", "imz": "HumanoidImZ, head and hands, latent policy + frozen decoder",
                "distill": "HumanoidImDistillGetup student, encoder 934 -> 1536-1024-512-160 -> 64, decoder 390 -> 3096-2048-1024 -> 69 SiLU"}[kind]
        line = {"workload": "evaluation pass (%s): %d envs, %d clips (median %d frames), no physics" % (name, n, args.clips, args.median_frames),
                "gpu": info, "passes": args.passes}
        for a, r in res.items():
            mean = sum(r["pass_s"]) / len(r["pass_s"])
            line[a] = {"pass_s": round(mean, 4), "pass_s_min_max": [round(min(r["pass_s"]), 4), round(max(r["pass_s"]), 4)],
                       "chunks": r["chunks"], "steps": r["steps"], "eval_env_steps_per_s": round(n * r["steps"] / mean, 1),
                       "eval_steps_per_s": round(r["steps"] / mean, 1),
                       "chunk_load_ms": round(1e3 * sum(r["load_s"]) / len(r["load_s"]), 3),
                       "chunk_readback_ms": round(1e3 * sum(r["read_s"]) / len(r["read_s"]), 3)}
        line["eager_over_graph"] = round(line["eager"]["pass_s"] / line["graph"]["pass_s"], 2)
        if kind == "distill":
            mac = student_macs(d.vae)
            line["gemm_mac_per_env"] = mac
            line["gemm_gflop_per_eval_step"] = round(2 * mac * n / 1e9, 3)
            for a in ("graph", "eager"):
                line[a]["gemm_tflops"] = round(2 * mac * n * line[a]["eval_steps_per_s"] / 1e12, 2)
            ms = student_step_ms(d)
            line["student_ms_per_step"] = round(ms, 4)                     # encoder + Z_MEAN + decoder + PD targets, alone, in graphs
            line["student_tflops"] = round(2 * mac * n / ms / 1e9, 1)
            line["student_share_of_graph_pass"] = round(ms * line["graph"]["steps"] / 1e3 / line["graph"]["pass_s"], 3)
        print(json.dumps(line), flush=True)
        if i == 0:
            step_s, metrics_s = reference_path(d, ds, args.ref_steps)
            print(json.dumps({"workload": "reference per-step path: MotionLib query + .cpu() of body_pos and body_pos_gt, %d envs, %d steps; "
                                          "compute_metrics_lite (numpy) over the %d sequences" % (n, args.ref_steps, n), "gpu": info,
                              "step_ms": round(1e3 * step_s / args.ref_steps, 3), "steps_per_s": round(args.ref_steps / step_s, 1),
                              "compute_metrics_lite_s": round(metrics_s, 3)}), flush=True)
        del d
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
