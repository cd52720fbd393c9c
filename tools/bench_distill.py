#!/usr/bin/env python
"""Full PULSE distillation iterations on the device (`DistillStepsB200`): one horizon of HumanoidImDistillGetup (getup resets inside the
horizon, frozen teacher, VAE student, pre-physics and step kernels; no physics) followed by the only_kin_loss update (6 mini-epochs of
16384-row minibatches), on synthetic MotionLib tables and simulator state (tools/synth.py).

  sizes   8192 envs (config C3) and 16384 envs, horizon 32
  nets    im_z_fit.yaml widths for the student, the env_im_vae.yaml teacher (3 x (1024, 512) ReLU columns + (1024, 512) SiLU composer)
  getup   recovery 0.3, fall 0.1 (env_im_vae.yaml), 60 recovery steps, a fall pool of n random states

Per size, one JSON line: the card name, power limit and maximum SM clock read in the same run; horizon and update milliseconds from device
events (means over --iters iterations after --warmup); env-steps/s of the whole iteration; the same horizon with the teacher on the main
stream, alternated iteration by iteration with the side-stream schedule; and the reset-class counts (reference-state, fall, recovery) of
one further horizon, counted through a refresh hook (which runs that horizon as graph segments).  Needs a CUDA device: there is no fallback.

  python tools/bench_distill.py [--envs 8192 16384] [--iters 5] [--warmup 2]
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
P_REC, P_FALL, REC_STEPS = 0.3, 0.1, 60


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception:
        return "unknown"


def build(n, dev):
    from pulse_b200.distill import DistillStepsB200
    from pulse_b200.humanoid_im import HumanoidImCompute
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.vae import PulseVAE, TeacherPNN
    from tools.synth import device_step_inputs, device_tables
    ml = MotionLibB200.from_tables(device_tables(n, dev, seed=100, median_frames=150))
    z = device_step_inputs(ml, n, seed=200)
    comp = HumanoidImCompute(ml)
    root = torch.zeros(n, 2, 13, device=dev)
    root[:, 0] = z["body_state"][:, 0]
    sim = dict(body_state=z["body_state"], root_states=root[:, 0], dof_pos=z["dof_pos"], dof_vel=z["dof_vel"], dof_force=z["dof_force"],
               progress_buf=z["progress_buf"], motion_ids=z["motion_ids"], motion_start_times=z["motion_start_times"],
               motion_start_offset=z["motion_start_offset"], global_offset=z["global_offset"], cycle_counter=z["cycle_counter"],
               contact_forces=torch.zeros(n, 24, 3, device=dev), actor_ids=torch.arange(n, dtype=torch.int32, device=dev))
    g = torch.Generator(device=dev).manual_seed(300)
    fall_dof = torch.randn(n, 69, 2, device=dev, generator=g)
    getup = dict(recovery_counter=torch.zeros(n, dtype=torch.int32, device=dev), available_fall_states=torch.zeros(n, dtype=torch.long, device=dev),
                 fall_id_assignments=torch.zeros(n, dtype=torch.long, device=dev), fall_root_states=torch.randn(n, 13, device=dev, generator=g),
                 fall_dof_pos=fall_dof[..., 0], fall_dof_vel=fall_dof[..., 1], recovery_prob=P_REC, fall_prob=P_FALL, recovery_steps=REC_STEPS)
    vae = PulseVAE(device=dev, horizon=HORIZON, with_critic=False)
    teacher = TeacherPNN(device=dev, prim_units=(1024, 512), composer_units=(1024, 512), num_prim=3)
    drv = DistillStepsB200(comp, vae, teacher, sim, getup, horizon=HORIZON, reset_seed=1)
    drv.first_observation()
    return drv


def timed(fn, dev):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    return s, e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[8192, 16384])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_distill.py needs a CUDA device")
    dev = "cuda:0"
    info = gpu_info()
    for n in args.envs:
        drv = build(n, dev)
        ev = {"side": [], "main": [], "update": []}
        epoch = 0
        for it in range(args.warmup + args.iters):
            for sched in ("side", "main"):             # the two schedules alternate, so both see the same conditions
                drv.teacher_side = sched == "side"
                h = timed(drv.play_steps, dev)
                u = timed(lambda: drv.train_epoch(epoch, mini_epochs=MINI_EPOCHS, minibatch=MINIBATCH), dev)
                epoch += 1
                if it >= args.warmup:
                    ev[sched].append(h)
                    ev["update"].append(u)
        torch.cuda.synchronize()
        ms = {k: sum(s.elapsed_time(e) for s, e in v) / len(v) for k, v in ev.items()}
        drv.teacher_side = True
        counts = torch.zeros(3, dtype=torch.int64, device=dev)
        drv.refresh = lambda t, ws: counts.add_(ws["class_counts"])
        drv.play_steps(check=True)
        drv.refresh = None
        torch.cuda.synchronize()
        c = counts.tolist()
        L = drv.vae.losses(MINIBATCH)
        print(json.dumps({
            "workload": "PULSE distillation iteration (HumanoidImDistillGetup, only_kin_loss): %d envs, horizon %d, im_z_fit.yaml student, "
                        "env_im_vae.yaml teacher, %d mini-epochs of %d rows, no physics" % (n, HORIZON, MINI_EPOCHS, MINIBATCH),
            "gpu": info, "envs": n, "horizon_ms": round(ms["side"], 3), "update_ms": round(ms["update"], 3),
            "env_steps_per_s": round(n * HORIZON / ((ms["side"] + ms["update"]) * 1e-3), 1),
            "horizon_ms_teacher_on_main_stream": round(ms["main"], 3),
            "resets_per_horizon": {"reference_state": c[0], "fall": c[1], "recovery": c[2]},
            "kin_loss_last_minibatch": round(L["kin_loss"], 5), "iters": args.iters, "warmup": args.warmup}), flush=True)
        del drv
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
