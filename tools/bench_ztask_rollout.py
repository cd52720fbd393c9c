#!/usr/bin/env python
"""Full training iterations of a latent-space task on the device (`ZTaskStepsB200`, BASELINE config C5): one horizon of HumanoidReachZ /
HumanoidSpeedZ / HumanoidStrikeZ (device resets inside the horizon, latent policy 2048-1024-512 SiLU, frozen PULSE prior + decoder,
pre-physics and step kernels; no physics), then `finish` and the PPO update (6 mini-epochs of 16384-row minibatches), on synthetic
MotionLib tables and simulator state (tools/synth.py).  One env in 16 starts below its termination height with a contact force and the
progress counters are spread over the episode length, so envs reset in every horizon.

Two arms, alternated iteration by iteration in the same call so both see the same conditions:
  graph   the driver as shipped: the horizon is one CUDA graph over four streams, one graph per update minibatch
  eager   the same entry points with use_graphs=False: one stream, every launch issued from the host
--policy picks the policy: latent (the default, above), direct (the PPO baseline HumanoidReach / HumanoidSpeed / HumanoidStrike under
learning=ppo: ZTaskStepsB200 with vae=None, the same 2048-1024-512 SiLU network acting in the 69 dofs with sigma exp(-2.9), no prior
or decoder), or both (the latent and the direct drivers' graph and eager arms alternated iteration by iteration, on MotionLib tables
and simulator state built from the same seeds).  One JSON line per size and policy.

Per size, one JSON line: the card name, power limit and maximum SM clock read in the same call; per arm the launches per step
(`pulse_launch_count` over one eager horizon / T; the graph arm replays the launches it captured, fork and join included), the
milliseconds per horizon and per update (device events; mean, min and max over --iters iterations after --warmup, with an L2 flush
before each timed region) and the env-steps/s of the rollout and of the full iteration.  Needs a CUDA device: there is no fallback.

  python tools/bench_ztask_rollout.py [--kind reach|speed|strike] [--policy latent|direct|both] [--envs 1024 8192] [--iters 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HORIZON, MINIBATCH, MINI_EPOCHS = 32, 16384, 6
UNITS = (2048, 1024, 512)          # pulse_z_task.yaml:27-28 and ppo.yaml
POLICIES = {"latent": ("latent",), "direct": ("direct",), "both": ("latent", "direct")}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def build(kind, n, dev, use_graphs, policy="latent"):
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.reach import ReachTaskB200
    from pulse_b200.vae import PulseVAE
    from pulse_b200.ztask_reset import ZTaskResetB200
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    from pulse_b200.ztasks import SpeedTaskB200, StrikeTaskB200
    from tools.synth import device_step_inputs, device_tables
    tables = device_tables(min(n, 2048), dev, seed=100, median_frames=150)
    ml = MotionLibB200.from_tables(tables)
    g = torch.Generator(device=dev).manual_seed(300)
    floor = -0.9 + 0.05 * torch.rand(tables["gts"].shape[0], device=dev, generator=g)      # stand-in for the SMPL ground table
    z = device_step_inputs(ml, n, seed=200, bodies_per_env=26, dofs_per_env=72)
    body, contact = z["body_state"], torch.zeros(n, 26, 3, device=dev)
    body[::16, 5, 2], contact[::16, 5, 2] = 0.05, 5.0                                       # fallen: reset at the second step
    root = torch.zeros(n, 2, 13, device=dev)
    root[:, 0] = body[:, 0]
    root[:, 1, 0:3] = torch.randn(n, 3, device=dev, generator=g)
    root[:, 1, 6] = 1.0
    sim = dict(body_state=body, root_states=root[:, 0], dof_pos=z["dof_pos"], dof_vel=z["dof_vel"],
               progress_buf=torch.randint(2, 300, (n,), device=dev, generator=g), sampled_motion_ids=z["motion_ids"].clone(),
               motion_start_times=z["motion_start_times"], contact_forces=contact, actor_ids=torch.arange(n, dtype=torch.int32, device=dev) * 2)
    if kind == "strike":
        sim.update(target_states=root[:, 1], tar_contact_forces=torch.zeros(n, 3, device=dev), tar_actor_ids=sim["actor_ids"] + 1)
    task = {"reach": ReachTaskB200, "speed": SpeedTaskB200, "strike": StrikeTaskB200}[kind](n, device=dev)
    if policy == "direct":                                                                  # ppo.yaml: the policy writes the 69 dof targets
        pol, vae = PPOPolicy(obs_size=task.obs_size, num_actions=69, units=UNITS, act="silu", logstd=-2.9, device=dev, seed=0), None
    else:
        pol = PPOPolicy(obs_size=task.obs_size, num_actions=32, units=UNITS, act="silu", device=dev, seed=0)
        vae = PulseVAE(device=dev, with_critic=False)                                       # the frozen prior + decoder
    drv = ZTaskStepsB200(task, ZTaskResetB200(kind, ml, floor), pol, vae, sim, horizon=HORIZON, use_graphs=use_graphs, reset_seed=1)
    drv.first_observation()
    return drv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", choices=("reach", "speed", "strike"), default="reach")
    ap.add_argument("--policy", choices=tuple(POLICIES), default="latent")
    ap.add_argument("--envs", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if args.iters < 3:
        raise SystemExit("at least three timed iterations")
    if not torch.cuda.is_available():
        raise SystemExit("bench_ztask_rollout.py needs a CUDA device")
    from pulse_b200 import _lib
    lib = _lib.load()
    dev = "cuda:0"
    info = gpu_info()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)                  # larger than the 50 MB L2

    def timed(fn):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        return s, e

    for n in args.envs:
        pols = POLICIES[args.policy]
        arms = {(pol, mode): build(args.kind, n, dev, mode == "graph", pol) for pol in pols for mode in ("graph", "eager")}
        mb = min(MINIBATCH, n * HORIZON)
        update = lambda d: (d.finish(), d.train_epoch(mini_epochs=MINI_EPOCHS, minibatch=mb))
        ev = {a: {"horizon": [], "update": []} for a in arms}
        resets = {a: 0.0 for a in arms}
        for it in range(args.warmup + args.iters):                 # warm-up covers the eager run and the capture of every graph
            for a, d in arms.items():
                h = timed(d.play_steps)
                done = d.dones.sum()
                u = timed(lambda: update(d))
                if it >= args.warmup:
                    ev[a]["horizon"].append(h)
                    ev[a]["update"].append(u)
                    resets[a] += float(done)
        torch.cuda.synchronize()
        launches = {}
        for pol in pols:
            c0 = lib.pulse_launch_count()
            arms[(pol, "eager")].play_steps()
            torch.cuda.synchronize()
            launches[pol] = (lib.pulse_launch_count() - c0) / HORIZON
        for pol in pols:
            what = ("latent-space %s task iteration (Humanoid%sZ, pulse_z_task.yaml): %d envs, horizon %d, latent policy %s SiLU, frozen prior + decoder"
                    if pol == "latent" else
                    "PPO baseline %s task iteration (Humanoid%s, ppo.yaml): %d envs, horizon %d, policy %s SiLU over the 69 dofs, no prior or decoder")
            out = {"workload": (what + ", task reward only, %d mini-epochs of %d rows, no physics, no discriminator")
                               % (args.kind, args.kind.capitalize(), n, HORIZON, "-".join(map(str, UNITS)), MINI_EPOCHS, mb),
                   "gpu": info, "kind": args.kind, "envs": n, "iters": args.iters, "warmup": args.warmup, "policy": pol,
                   "launches_per_step": round(launches[pol], 2)}
            for mode in ("graph", "eager"):
                a = (pol, mode)
                ms = {k: [s.elapsed_time(e) for s, e in v] for k, v in ev[a].items()}
                mean = {k: sum(v) / len(v) for k, v in ms.items()}
                out[mode] = {"horizon_ms": round(mean["horizon"], 3), "horizon_ms_min_max": [round(min(ms["horizon"]), 3), round(max(ms["horizon"]), 3)],
                             "update_ms": round(mean["update"], 3), "update_ms_min_max": [round(min(ms["update"]), 3), round(max(ms["update"]), 3)],
                             "rollout_env_steps_per_s": round(n * HORIZON / (mean["horizon"] * 1e-3), 1),
                             "iteration_env_steps_per_s": round(n * HORIZON / ((mean["horizon"] + mean["update"]) * 1e-3), 1),
                             "resets_per_horizon": round(resets[a] / args.iters, 1)}
            print(json.dumps(out), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
