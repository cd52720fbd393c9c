#!/usr/bin/env python
"""Full training iterations of the pedestrian terrain task on the device (`TerrainStepsB200`): one horizon of HumanoidPedestrianTerrainZ
(device resets inside the horizon, the amp_sept policy with its 512-256 task encoder and 2048-1024-512 SiLU actor and critic, frozen
PULSE prior + decoder, PD targets and the terrain step kernel; no physics), then `finish` and the PPO update (6 mini-epochs of
min(16384, n * 32)-row minibatches), on synthetic MotionLib tables and simulator state (tools/synth.py) over a 2000 x 5000 synthetic
heightfield with a walkable table of about 70 % of its cells (as tools/bench_terrain_reset.py builds them).  One env in 16 starts
with a contact force on a non-contact body and the progress counters are spread over the episode length, so envs reset in every
horizon.

Two arms, alternated iteration by iteration in the same call so both see the same conditions:
  graph   the driver as shipped: the horizon is one CUDA graph over four streams, one graph per update minibatch
  eager   the same entry points with use_graphs=False: one stream, every launch issued from the host

Per size, one JSON line: the card name, power limit and maximum SM clock read in the same call; per arm the launches per step
(`pulse_launch_count` over one eager horizon / T; the graph arm replays the launches it captured, fork and join included), the
milliseconds per horizon and per update (device events; mean, min and max over --iters iterations after --warmup, with an L2 flush
before each timed region), the env-steps/s of the rollout and of the full iteration, and the resets per horizon.  Needs a CUDA
device: there is no fallback.

  python tools/bench_terrain_rollout.py [--envs 1536 8192] [--iters 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HORIZON, MINIBATCH, MINI_EPOCHS = 32, 16384, 6
ROWS, COLS, HSCALE = 2000, 5000, 0.1


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def terrain_tables(dev):
    """The heightfield (steps of 0.2 m every 5 m of x plus noise) and its walkable table (the cells inside a 5 m border, 70 % of them)."""
    from pulse_b200.terrain import TerrainB200
    from tests import terrain_reset_oracle as tro
    rng = np.random.default_rng(0)
    hf = torch.from_numpy((rng.integers(0, 40, size=(ROWS, COLS)) + (np.arange(ROWS)[:, None] // 50 % 4) * 40).astype(np.int16))
    walk = torch.from_numpy((rng.random((ROWS, COLS)) < 0.3).astype(np.int16))
    cx, cy = tro.walkable_table(walk, HSCALE, 50)
    return TerrainB200(hf, horizontal_scale=HSCALE, device=dev), cx, cy


def build(n, dev, use_graphs, terrain, cx, cy):
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.sept import SeptPolicy
    from pulse_b200.terrain import PedestrianTerrainTaskB200
    from pulse_b200.terrain_reset import TerrainResetB200
    from pulse_b200.terrain_rollout import TerrainStepsB200
    from pulse_b200.vae import PulseVAE
    from tools.synth import device_step_inputs, device_tables
    tables = device_tables(min(n, 2048), dev, seed=100, median_frames=150)
    ml = MotionLibB200.from_tables(tables)
    g = torch.Generator(device=dev).manual_seed(300)
    floor = -0.9 + 0.05 * torch.rand(tables["gts"].shape[0], device=dev, generator=g)      # stand-in for the SMPL ground table
    z = device_step_inputs(ml, n, seed=200, bodies_per_env=26, dofs_per_env=72)
    body, contact = z["body_state"], torch.zeros(n, 26, 3, device=dev)
    i = torch.randint(0, cx.shape[0], (n,), device=dev, generator=g)
    spawn = torch.stack([cx.to(dev)[i], cy.to(dev)[i]], dim=-1)
    body[..., 0:2] += (spawn - body[:, 0, 0:2])[:, None]                                     # every humanoid on a walkable cell
    contact[::16, 5, 2] = 60.0                                                                # fallen: reset at the next step
    root = torch.zeros(n, 2, 13, device=dev)
    root[:, 0] = body[:, 0]
    root[:, 1, 6] = 1.0
    sim = dict(body_state=body, root_states=root[:, 0], dof_pos=z["dof_pos"], dof_vel=z["dof_vel"],
               progress_buf=torch.randint(2, 300, (n,), device=dev, generator=g), sampled_motion_ids=z["motion_ids"].clone(),
               motion_start_times=z["motion_start_times"], contact_forces=contact, actor_ids=torch.arange(n, dtype=torch.int32, device=dev) * 2)
    task = PedestrianTerrainTaskB200(n, device=dev, terrain=terrain)
    task.reset_task(torch.arange(n, device=dev), sim["root_states"])
    policy = SeptPolicy(num_actions=32, with_disc=False, device=dev, seed=0)                 # pulse_z_terrain.yaml's amp_sept network
    vae = PulseVAE(device=dev, with_critic=False)                                           # the frozen prior + decoder
    drv = TerrainStepsB200(task, TerrainResetB200(ml, floor, terrain, cx, cy), policy, vae, sim, horizon=HORIZON, use_graphs=use_graphs,
                           reset_seed=1)
    drv.first_observation()
    return drv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[1536, 8192])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if args.iters < 3:
        raise SystemExit("at least three timed iterations")
    if not torch.cuda.is_available():
        raise SystemExit("bench_terrain_rollout.py needs a CUDA device")
    from pulse_b200 import _lib
    lib = _lib.load()
    dev = "cuda:0"
    info = gpu_info()
    terrain, cx, cy = terrain_tables(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)                  # larger than the 50 MB L2

    def timed(fn):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        return s, e

    for n in args.envs:
        arms = {"graph": build(n, dev, True, terrain, cx, cy), "eager": build(n, dev, False, terrain, cx, cy)}
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
        c0 = lib.pulse_launch_count()
        arms["eager"].play_steps()
        torch.cuda.synchronize()
        launches = (lib.pulse_launch_count() - c0) / HORIZON
        out = {"workload": "pedestrian terrain task iteration (HumanoidPedestrianTerrainZ, pulse_z_terrain.yaml): %d envs, horizon %d, "
                           "amp_sept policy (task encoder 512-256, actor / critic 2048-1024-512 SiLU), frozen prior + decoder, task reward only, "
                           "%d mini-epochs of %d rows, %d x %d heightfield, no physics, no discriminator" % (n, HORIZON, MINI_EPOCHS, mb, ROWS, COLS),
               "gpu": info, "envs": n, "iters": args.iters, "warmup": args.warmup, "launches_per_step": round(launches, 2)}
        for a in arms:
            ms = {k: [s.elapsed_time(e) for s, e in v] for k, v in ev[a].items()}
            mean = {k: sum(v) / len(v) for k, v in ms.items()}
            out[a] = {"horizon_ms": round(mean["horizon"], 3), "horizon_ms_min_max": [round(min(ms["horizon"]), 3), round(max(ms["horizon"]), 3)],
                      "update_ms": round(mean["update"], 3), "update_ms_min_max": [round(min(ms["update"]), 3), round(max(ms["update"]), 3)],
                      "rollout_env_steps_per_s": round(n * HORIZON / (mean["horizon"] * 1e-3), 1),
                      "iteration_env_steps_per_s": round(n * HORIZON / ((mean["horizon"] + mean["update"]) * 1e-3), 1),
                      "resets_per_horizon": round(resets[a] / args.iters, 1)}
        print(json.dumps(out), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
