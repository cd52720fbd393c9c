#!/usr/bin/env python
"""Per-call time of the latent-space tasks' reset at 16384 envs: `pulse_reset_ztask` (Philox draws, 10 AMP history rows of 195
floats) and, for reach and speed, `pulse_ztask_reset_task`, for 5 % and 100 % of the envs resetting in mask mode.

Device events around each call, after warm-up, averaged over --calls calls.  The simulator refresh and the observation of the reset
envs are not part of the call.  Prints one JSON line per (task, fraction) with the card name, power limit and maximum SM clock read in
the same run.  Needs a CUDA device: there is no fallback.

  python tools/bench_ztask_reset.py [--envs 16384] [--calls 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ztask_reset.py needs a CUDA device")
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ztask_reset import ZTaskResetB200, smpl_ground_table
    from tests import ztask_reset_oracle as zo
    from tests.helpers import exact_tables

    dev, n = "cuda:0", args.envs
    tb = exact_tables(200, seed=3)
    keys = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames", "dt", "length_starts")
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in keys}, device=dev)
    floor = smpl_ground_table(tb.motion_aa, zo.StandInParser(), torch.linspace(-1.0, 1.0, 10)).to(dev)
    g = torch.Generator().manual_seed(0)
    root = torch.zeros(n, 2, 13, device=dev)
    dof = torch.zeros(n, 72, 2, device=dev)
    body = torch.zeros(n, 26, 13, device=dev)
    contact = torch.zeros(n, 26, 3, device=dev)
    amp = torch.zeros(n, 10, 195, device=dev)
    progress, terminate = torch.zeros(n, dtype=torch.int64, device=dev), torch.zeros(n, dtype=torch.int64, device=dev)
    mids, t0 = torch.zeros(n, dtype=torch.int64, device=dev), torch.zeros(n, device=dev)
    reset_buf = torch.zeros(n, dtype=torch.int64, device=dev)
    actors = torch.arange(n, dtype=torch.int32, device=dev) * 2
    tar_pos, tar_speed, change = torch.zeros(n, 3, device=dev), torch.zeros(n, device=dev), torch.zeros(n, dtype=torch.int64, device=dev)
    info = gpu_info()
    for kind in ("reach", "speed", "strike"):
        r = ZTaskResetB200(kind, ml, floor)
        for frac in (0.05, 1.0):
            mask = (torch.rand(n, generator=g) < frac).long().to(dev)

            def call(i):
                reset_buf.copy_(mask)
                r.reset_envs(root_states=root[:, 0], dof_pos=dof[:, :69, 0], dof_vel=dof[:, :69, 1], rigid_body_state=body, progress_buf=progress,
                             sampled_motion_ids=mids, motion_start_times=t0, reset_buf=reset_buf, terminate_buf=terminate, contact_forces=contact,
                             amp_obs_buf=amp, actor_ids=actors, target_states=root[:, 1] if kind == "strike" else None, tar_actor_ids=actors + 1,
                             seed=1, offset=i)
                if kind == "reach":
                    r.reset_task(progress_buf=progress, change_steps=change, tar_pos=tar_pos, seed=1, offset=i)
                elif kind == "speed":
                    r.reset_task(progress_buf=progress, change_steps=change, tar_speed=tar_speed, seed=1, offset=i)

            for i in range(args.warmup):
                call(i)
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for i in range(args.calls):
                call(args.warmup + i)
            e.record()
            torch.cuda.synchronize()
            print(json.dumps({"task": kind, "envs": n, "reset_fraction": frac, "reset_envs": int(mask.sum()), "gpu": info,
                              "us_per_call": round(1000.0 * s.elapsed_time(e) / args.calls, 1)}), flush=True)


if __name__ == "__main__":
    main()
