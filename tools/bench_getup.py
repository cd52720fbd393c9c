#!/usr/bin/env python
"""Per-call time of HumanoidImGetup's reset at 16384 envs, device path against the reference-style path.

  device     pulse_reset_getup (Philox draws) + the observation launch over the reset envs + pulse_getup_amp_init: no host round trip
  reference  the oracle composite of tests/getup_oracle.py on CUDA tensors -- `_reset_actors` with its Bernoulli masks, boolean
             indexing, nonzero and randperm, the reference-state reset, observation and AMP initialisation -- which synchronises with
             the host the way the reference's path does

For 5 %, 13 % and 50 % of the envs resetting (recoveryEpisodeProb 0.3, fallInitProb 0.1 as in env_im_vae.yaml, 30 % of the reset envs
terminated): device events around each call, after warm-up, averaged over --calls calls.  The simulator refresh between the reset and
the AMP initialisation is not part of either path.  Prints one JSON line per fraction with the card name, power limit and maximum SM
clock read in the same run.  Needs a CUDA device: there is no fallback.

  python tools/bench_getup.py [--envs 16384] [--calls 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

P_REC, P_FALL, STEPS = 0.3, 0.1, 60


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
        raise SystemExit("bench_getup.py needs a CUDA device")
    from oracle import pulse_oracle as po
    from pulse_b200 import _lib
    from pulse_b200.humanoid_im import HumanoidImCompute
    from pulse_b200.motion_lib import MotionLibB200
    from tests import getup_oracle as go
    from tests.helpers import exact_step_inputs, exact_tables

    dev, n = "cuda:0", args.envs
    tb = exact_tables(200, seed=3)
    z, _ = exact_step_inputs(tb, n, seed=4)
    keys = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames", "dt", "length_starts")
    comp = HumanoidImCompute(MotionLibB200.from_tables({k: getattr(tb, k) for k in keys}, device=dev))
    tb_dev = po.MotionTables(**{f: getattr(tb, f).to(dev) for f in tb.__dataclass_fields__})
    g = torch.Generator().manual_seed(0)
    st = {"motion_ids": z["motion_ids"], "start_times": z["start_times"], "start_offset": z["start_offset"], "global_offset": z["global_offset"],
          "cycle_counter": z["cycle_counter"], "progress_buf": z["progress_buf"], "root_states": torch.randn(n, 13, generator=g),
          "dof_pos": z["dof_pos"], "dof_vel": z["dof_vel"], "body_state": z["body_state"], "contact_forces": torch.zeros(n, 24, 3),
          "amp_obs_buf": torch.zeros(n, 10, 196), "obs_buf": torch.zeros(n, 934), "dof_force": z["dof_force"],
          "reset_buf": torch.zeros(n, dtype=torch.long), "terminate_buf": torch.zeros(n, dtype=torch.long),
          "recovery_counter": torch.zeros(n, dtype=torch.int32), "avail": torch.zeros(n, dtype=torch.long), "fid": torch.zeros(n, dtype=torch.long),
          "fall_root": torch.randn(n, 13, generator=g), "fall_dof_pos": torch.randn(n, 69, generator=g), "fall_dof_vel": torch.zeros(n, 69)}
    st = {k: v.to(dev) for k, v in st.items()}
    info = gpu_info()
    for frac in (0.05, 0.13, 0.5):
        mask = (torch.rand(n, generator=g) < frac).to(dev)
        term = (torch.rand(n, generator=g) < 0.3).long().to(dev)
        d = {k: v.clone() for k, v in st.items()}
        body = d["body_state"]

        def device_call(i):
            d["reset_buf"].copy_(mask.long())
            d["terminate_buf"].copy_(term)
            ws = comp.reset_getup(motion_ids=d["motion_ids"], motion_start_times=d["start_times"], motion_start_offset=d["start_offset"],
                                  global_offset=d["global_offset"], progress_buf=d["progress_buf"], root_states=d["root_states"],
                                  dof_pos=d["dof_pos"], dof_vel=d["dof_vel"], rigid_body_state=body, reset_buf=d["reset_buf"],
                                  terminate_buf=d["terminate_buf"], cycle_counter=d["cycle_counter"], contact_forces=d["contact_forces"],
                                  amp_obs_buf=d["amp_obs_buf"], recovery_counter=d["recovery_counter"], available_fall_states=d["avail"],
                                  fall_id_assignments=d["fid"], fall_root_states=d["fall_root"], fall_dof_pos=d["fall_dof_pos"],
                                  fall_dof_vel=d["fall_dof_vel"], recovery_prob=P_REC, fall_prob=P_FALL, recovery_steps=STEPS, seed=1, offset=i)
            comp.step(body_state=body, progress_buf=d["progress_buf"], motion_ids=d["motion_ids"], motion_start_times=d["start_times"],
                      motion_start_offset=d["start_offset"], global_offset=d["global_offset"], obs_buf=d["obs_buf"], env_ids=ws["env_list"],
                      env_count=ws["count"], flags=_lib.STEP_OBS)
            comp.getup_amp_init(body_state=body, dof_pos=d["dof_pos"], dof_vel=d["dof_vel"], amp_obs_buf=d["amp_obs_buf"])

        r = {k: v.clone() for k, v in st.items()}

        def reference_call(i):
            nonlocal r
            r["terminate_buf"].copy_(term)
            with torch.device(dev):            # the oracle's own constants (distances, index lists) on the GPU too
                ids = mask.nonzero().flatten()
                u = torch.rand(3, n)
                out, inf = go.getup_reset(tb_dev, po.ImStepConfig(), r, ids, u[0], u[1], u[2], torch.rand(n), P_REC, P_FALL, STEPS)
                out["amp_obs_buf"] = go.getup_amp_init(out["amp_obs_buf"], out["body_state"], out["dof_pos"], out["dof_vel"], inf["fall_ids"],
                                                       inf["recovery_ids"])
            r = out

        res = {"envs": n, "reset_fraction": frac, "gpu": info}
        for name, fn in (("device", device_call), ("reference", reference_call)):
            for i in range(args.warmup):
                fn(i)
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for i in range(args.calls):
                fn(args.warmup + i)
            e.record()
            torch.cuda.synchronize()
            res[f"{name}_us_per_call"] = round(1000.0 * s.elapsed_time(e) / args.calls, 1)
        res["speedup"] = round(res["reference_us_per_call"] / res["device_us_per_call"], 1)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
