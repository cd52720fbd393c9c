#!/usr/bin/env python
"""Per-call time of the pedestrian terrain task's reset at 16384 envs, for 5 % and 100 % of the envs resetting (mask mode), on a
2000 x 5000 heightfield (the env_pulse_terrain map of DESIGN.md section 3.9) with a walkable table of about 70 % of its cells.

  device arm  `pulse_reset_terrain` (Philox draws, 10 AMP history rows of 196 floats) + the list observation of the reset envs
              (`pulse_terrain_step`, PULSE_STEP_OBS) + `pulse_traj_reset_list`;
  oracle arm  the same composite as tensor operations on CUDA tensors (tests/terrain_reset_oracle.py and the oracle's observation and
              trajectory generator), with the reference's boolean-mask indexing and host location draw.

Device events around each call, after warm-up, averaged over --calls calls.  Prints one JSON line per fraction with the card name,
power limit and maximum SM clock read in the same run.  Needs a CUDA device: there is no fallback.

  python tools/bench_terrain_reset.py [--envs 16384] [--calls 30] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
from dataclasses import fields, replace

import numpy as np
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


def timed(fn, calls, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(calls):
        fn(warmup + i)
    e.record()
    torch.cuda.synchronize()
    return 1000.0 * s.elapsed_time(e) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_terrain_reset.py needs a CUDA device")
    from oracle import terrain_oracle as to
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.terrain import PedestrianTerrainTaskB200, TerrainB200
    from pulse_b200.terrain_reset import TerrainResetB200
    from pulse_b200.ztask_reset import smpl_ground_table
    from tests import terrain_reset_oracle as tro
    from tests import ztask_reset_oracle as zo
    from tests.helpers import exact_tables

    dev, n = "cuda:0", args.envs
    tb = exact_tables(200, seed=3)
    keys = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames", "dt", "length_starts")
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in keys}, device=dev)
    floor = smpl_ground_table(tb.motion_aa, zo.StandInParser(), torch.linspace(-1.0, 1.0, 10)).to(dev)
    rng = np.random.default_rng(0)
    rows, cols = 2000, 5000
    hf = torch.from_numpy((rng.integers(0, 40, size=(rows, cols)) + (np.arange(rows)[:, None] // 50 % 4) * 40).astype(np.int16))
    walk = torch.from_numpy((rng.random((rows, cols)) < 0.3).astype(np.int16))
    cx, cy = tro.walkable_table(walk, 0.1, 50)
    terrain = TerrainB200(hf, device=dev)
    r = TerrainResetB200(ml, floor, terrain, cx, cy)
    task = PedestrianTerrainTaskB200(n, device=dev, terrain=terrain, dt=zo.DT)
    root = torch.zeros(n, 2, 13, device=dev)
    root[:, 0, 6] = 1.0
    dof = torch.zeros(n, 72, 2, device=dev)
    body = torch.zeros(n, 26, 13, device=dev)
    contact = torch.zeros(n, 26, 3, device=dev)
    amp = torch.zeros(n, 10, 196, device=dev)
    progress, terminate = torch.zeros(n, dtype=torch.int64, device=dev), torch.zeros(n, dtype=torch.int64, device=dev)
    mids, t0 = torch.zeros(n, dtype=torch.int64, device=dev), torch.zeros(n, device=dev)
    reset_buf = torch.zeros(n, dtype=torch.int64, device=dev)
    actors = torch.arange(n, dtype=torch.int32, device=dev) * 2
    tb_dev = replace(tb, **{f.name: getattr(tb, f.name).to(dev) for f in fields(tb) if isinstance(getattr(tb, f.name), torch.Tensor)})
    hf_dev, cx_dev, cy_dev = hf.to(dev), cx.to(dev), cy.to(dev)
    prob = ml._sampling_batch_prob.to(dev)
    info = gpu_info()
    g = torch.Generator().manual_seed(0)
    for frac in (0.05, 1.0):
        mask = (torch.rand(n, generator=g) < frac).long().to(dev)

        def device_call(i):
            reset_buf.copy_(mask)
            r.reset_envs(root_states=root[:, 0], dof_pos=dof[:, :69, 0], dof_vel=dof[:, :69, 1], rigid_body_state=body, progress_buf=progress,
                         sampled_motion_ids=mids, motion_start_times=t0, reset_buf=reset_buf, terminate_buf=terminate, contact_forces=contact,
                         amp_obs_buf=amp, actor_ids=actors, seed=1, offset=i)
            r.observe(task, body, root[:, 0], progress)
            r.reset_task(task, root[:, 0], seed=2, offset=i)

        st = {"root_states": root[:, 0].clone(), "dof_pos": dof[:, :69, 0].clone(), "dof_vel": dof[:, :69, 1].clone(), "body_state": body[:, :24].clone(),
              "sampled_motion_ids": mids.clone(), "motion_start_times": t0.clone(), "progress_buf": progress.clone(), "reset_buf": mask.clone(),
              "terminate_buf": terminate.clone(), "contact_forces": contact[:, :24].clone(), "amp_obs_buf": amp.clone()}
        verts = task.traj_verts.clone()

        def oracle_call(i):
            ids = mask.nonzero().flatten()                      # the reference's boolean-mask indexing (a host read of the count)
            m = ids.numel()
            draws = {"motion_ids": torch.zeros(n, dtype=torch.int64, device=dev), "phase": torch.zeros(n, device=dev),
                     "loc_ids": torch.zeros(n, dtype=torch.int64, device=dev)}
            draws["motion_ids"][ids] = torch.multinomial(prob, m, replacement=True)
            draws["phase"][ids] = torch.rand(m, device=dev)
            draws["loc_ids"][ids] = torch.from_numpy(np.random.randint(0, cx.shape[0], size=m)).to(dev)
            o = tro.terrain_reset(tb_dev, st, ids, draws, floor, hf_dev, cx_dev, cy_dev, center_pts=to.center_height_points().to(dev))
            bs, rs = o["body_state"][ids], o["root_states"][ids]
            to.terrain_self_obs(hf_dev, 0.1, 0.005, bs, to.center_height_points().to(dev), True)
            samples = to.fetch_traj_samples(verts[ids], o["progress_buf"][ids], zo.DT, tro.TRAJ_DT)
            to.terrain_task_obs(hf_dev, 0.1, 0.005, rs, bs[:, to.HEAD_BODY_ID, 0:7], samples, to.square_height_points().to(dev),
                                to.center_height_points().to(dev), True)
            tro.reset_task(verts, ids, o["root_states"], torch.rand(n, to.TRAJ_DRAWS, device=dev))

        line = {"envs": n, "reset_fraction": frac, "reset_envs": int(mask.sum()), "heightfield": [rows, cols], "walkable": int(cx.shape[0]),
                "gpu": info, "device_us_per_call": round(timed(device_call, args.calls, args.warmup), 1)}
        try:
            with torch.device(dev):                             # the oracle's own arange / zeros on the device too
                line["oracle_us_per_call"] = round(timed(oracle_call, max(3, args.calls // 10), 1), 1)
        except Exception as exc:                                # reported, not hidden: the device arm's number stands on its own
            line["oracle_error"] = f"{type(exc).__name__}: {exc}"[:300]
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
