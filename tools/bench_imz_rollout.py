#!/usr/bin/env python
"""Full training iterations of the VR controller task on the device (`ImZStepsB200`): one horizon of HumanoidImZ (pulse_z_vr.yaml: head
and hands tracked, v6 observation of 430 floats, device resets inside the horizon, latent policy 2048-1536-1024-1024-512-512 SiLU, frozen
PULSE prior + decoder, tracked step kernel; no physics), then `finish` and the PPO update (6 mini-epochs of 16384-row minibatches), on
synthetic MotionLib tables and simulator state (tools/synth.py).  One env in 16 is displaced by 1 m (early termination) and the
progress counters are spread over the clips, so envs reset in every horizon.

Two arms, alternated iteration by iteration in the same call so both see the same conditions:
  graph   the driver as shipped: the horizon is one CUDA graph over four streams, one graph per update minibatch
  eager   the same entry points with use_graphs=False: one stream, every launch issued from the host
Per size, one JSON line: the card name, power limit and maximum SM clock read in the same call; per arm the launches per step, the
milliseconds per horizon and per update (device events; mean, min and max over --iters iterations after --warmup, with an L2 flush
before each timed region) and the env-steps/s of the rollout and of the full iteration.

Then one JSON line comparing the step at --kernel-envs envs (device events around --kernel-reps launches, the two arms alternated):
  track     pulse_im_track_step (v6, head and hands): reward, reset and the 430-float row in one launch
  general   HumanoidImB200Mixin's path for the same configuration: the fused step with the observation off, the fused step in
            observation mode into a 934-float scratch row (self observation), the MotionLib query and pulse_im_task_obs, and the two
            copies that assemble the row
Needs a CUDA device: there is no fallback.

  python tools/bench_imz_rollout.py [--envs 3072 8192] [--iters 5] [--warmup 2] [--kernel-envs 16384] [--kernel-reps 50]
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
UNITS = (2048, 1536, 1024, 1024, 512, 512)         # pulse_z_vr.yaml
VR = (13, 18, 23)                                  # env_pulse_im.yaml trackBodies: Head, L_Hand, R_Hand


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def make_state(n, dev):
    from pulse_b200.motion_lib import MotionLibB200
    from tools.synth import device_step_inputs, device_tables
    ml = MotionLibB200.from_tables(device_tables(min(n, 2048), dev, seed=100, median_frames=150))
    z = device_step_inputs(ml, n, seed=200, bodies_per_env=26, dofs_per_env=72)
    g = torch.Generator(device=dev).manual_seed(300)
    body = z["body_state"]
    body[::16, :, 0:3] += 1.0                                                               # displaced: early termination
    root = torch.zeros(n, 2, 13, device=dev)
    root[:, 0] = body[:, 0]
    root[:, 1, 6] = 1.0
    z["progress_buf"].copy_(torch.randint(2, 150, (n,), device=dev, generator=g))
    sim = dict(body_state=body, root_states=root[:, 0], dof_pos=z["dof_pos"], dof_vel=z["dof_vel"], progress_buf=z["progress_buf"],
               motion_ids=z["motion_ids"].clone(), motion_start_times=z["motion_start_times"], motion_start_offset=z["motion_start_offset"],
               global_offset=z["global_offset"], dof_force=z["dof_force"], contact_forces=torch.zeros(n, 26, 3, device=dev),
               actor_ids=torch.arange(n, dtype=torch.int32, device=dev) * 2)
    return ml, sim


def build(n, dev, use_graphs):
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    from pulse_b200.imz_rollout import ImZStepsB200
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.vae import PulseVAE
    ml, sim = make_state(n, dev)
    comp = HumanoidImCompute(ml, ImConfig(track_body_ids=VR))
    policy = PPOPolicy(obs_size=comp.obs_size, num_actions=32, units=UNITS, act="silu", logstd=-1.5, device=dev, seed=0)
    vae = PulseVAE(device=dev, with_critic=False)                                           # the frozen prior + decoder
    drv = ImZStepsB200(comp, policy, vae, sim, horizon=HORIZON, use_graphs=use_graphs, reset_seed=1)
    drv.first_observation()
    return drv


def bench_kernels(n, reps, dev, info):
    from pulse_b200 import _lib
    from pulse_b200.humanoid_im import IM_OBS, SELF_OBS, HumanoidImCompute, ImConfig
    ml, s = make_state(n, dev)
    full, tr = HumanoidImCompute(ml), HumanoidImCompute(ml, ImConfig(track_body_ids=VR))
    W = tr.obs_size
    kw = {k: s[k] for k in ("body_state", "motion_ids", "motion_start_times", "motion_start_offset", "global_offset", "dof_force", "dof_vel")}
    prog = s["progress_buf"]
    obs, scratch, self_obs, task = (torch.zeros(n, w, device=dev) for w in (W, IM_OBS, SELF_OBS, W - SELF_OBS))
    rew, raw = torch.zeros(n, device=dev), torch.zeros(n, 5, device=dev)
    reset, term = torch.zeros(n, dtype=torch.long, device=dev), torch.zeros(n, dtype=torch.long, device=dev)
    track_ids = torch.tensor(VR, dtype=torch.int32, device=dev)
    out = dict(rew_buf=rew, reward_raw=raw, reset_buf=reset, terminate_buf=term)

    def track():
        tr.step(flags=_lib.STEP_ALL, obs_buf=obs, progress_buf=prog, **out, **kw)

    def general():
        full.step(flags=_lib.STEP_REWARD | _lib.STEP_RESET, progress_buf=prog, **out, **kw)
        full.step(flags=_lib.STEP_OBS, obs_buf=scratch, self_obs_buf=self_obs, progress_buf=prog, **kw)
        full.task_obs(version=6, body_state=s["body_state"], progress_buf=prog, motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"],
                      motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"], track_ids=track_ids, obs_buf=task)
        obs[:, :SELF_OBS] = self_obs
        obs[:, SELF_OBS:] = task

    arms = {"track": track, "general": general}
    ms = {a: [] for a in arms}
    for a, fn in arms.items():                                     # warm-up: module loads, the MotionLib query's buffers
        fn()
    for _ in range(5):
        for a, fn in arms.items():
            s0, e0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for _ in range(reps):
                fn()
            e0.record()
            torch.cuda.synchronize()
            ms[a].append(s0.elapsed_time(e0) / reps)
    res = {"workload": "HumanoidImZ step (head and hands tracked, v6, %d floats): %d envs, power reward" % (W, n), "gpu": info, "envs": n,
           "reps": reps, "rounds": 5}
    for a in arms:
        v = ms[a]
        res[a + "_ms"] = round(sum(v) / len(v), 4)
        res[a + "_ms_min_max"] = [round(min(v), 4), round(max(v), 4)]
    res["general_over_track"] = round(res["general_ms"] / res["track_ms"], 2)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[3072, 8192])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--kernel-envs", type=int, default=16384)
    ap.add_argument("--kernel-reps", type=int, default=50)
    args = ap.parse_args()
    if args.iters < 3:
        raise SystemExit("at least three timed iterations")
    if not torch.cuda.is_available():
        raise SystemExit("bench_imz_rollout.py needs a CUDA device")
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
        arms = {"graph": build(n, dev, True), "eager": build(n, dev, False)}
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
        out = {"workload": "VR controller task iteration (HumanoidImZ, pulse_z_vr.yaml): %d envs, horizon %d, latent policy %s SiLU, frozen "
                           "prior + decoder, task reward only, %d mini-epochs of %d rows, no physics, no discriminator"
                           % (n, HORIZON, "-".join(map(str, UNITS)), MINI_EPOCHS, mb),
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
    bench_kernels(args.kernel_envs, args.kernel_reps, dev, info)


if __name__ == "__main__":
    main()
