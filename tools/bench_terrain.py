"""Kernel time of pulse_terrain_step (pedestrian terrain task: reward + reset + observation, one launch) at 16384 envs over an
env_pulse_terrain-sized heightfield (2000 x 5000 int16, 20 MB), timed with CUDA events around a CUDA graph of many launches.

  python tools/bench_terrain.py [--envs 16384] [--launches 200] [--reps 5] [--power]

Prints one JSON line: microseconds per launch and the algorithmic HBM rate against the H100 SXM's 3.35 TB/s.  The algorithmic bytes per
env-step are what the step must move at least once: body state 1248, actor root 52, contact forces 288, progress 8, trajectory
waypoints 264 (11 lookups x 2 waypoints x 12 B), observation 5608, reward + reward_raw 12, reset + terminate 16 (+ 552 for the power
term's dof force and velocity).  The heightfield reads (~4.2 KB per env: 1024 + 18 points x 2 int16 cells) are counted separately; the
20 MB map is expected to stay in the 50 MB L2.  Needs a CUDA device: there is no fallback.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_ENV = 1248 + 52 + 288 + 8 + 264 + 5608 + 12 + 16
POWER_BYTES_PER_ENV = 2 * 69 * 4
HF_BYTES_PER_ENV = (1024 + 2 * 9) * 2 * 2


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--power", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_terrain.py needs a CUDA device")
    from pulse_b200.terrain import PedestrianTerrainTaskB200, TerrainB200
    dev = "cuda:0"
    n = args.envs
    g = torch.Generator(device=dev).manual_seed(0)
    hf = torch.randint(-200, 400, (2000, 5000), generator=g, device=dev, dtype=torch.int16)
    task = PedestrianTerrainTaskB200(n, dev, TerrainB200(hf, device=dev), power_reward=args.power)
    rb = torch.zeros(n, 24, 13, device=dev)
    root = torch.rand(n, 3, generator=g, device=dev) * torch.tensor([190.0, 490.0, 0.5], device=dev) + torch.tensor([5.0, 5.0, 0.8], device=dev)
    rb[..., 0:3] = root[:, None] + 0.3 * torch.randn(n, 24, 3, generator=g, device=dev)
    rb[:, 0, 0:3] = root
    rb[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 24, 4, generator=g, device=dev), dim=-1)
    rb[..., 7:13] = torch.randn(n, 24, 6, generator=g, device=dev)
    roots = rb[:, 0].clone()
    prog = torch.randint(0, 300, (n,), generator=g, device=dev)
    cf = 20 * torch.randn(n, 24, 3, generator=g, device=dev)
    df, dv = torch.randn(n, 69, generator=g, device=dev), torch.randn(n, 69, generator=g, device=dev)
    task.reset_task(torch.arange(n, device=dev), root)
    step = lambda: task.post_physics_step(rb, roots, prog, cf, df, dv)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(args.launches):
            step()
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        graph.replay()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / args.launches)
    us = min(times)
    nbytes = n * (BYTES_PER_ENV + (POWER_BYTES_PER_ENV if args.power else 0))
    print(json.dumps({"kernel": "terrain_step_kernel", "envs": n, "power": args.power, "us_per_launch": round(us, 2),
                      "us_per_launch_all_reps": [round(t, 2) for t in times], "algorithmic_bytes": nbytes,
                      "algorithmic_GBps": round(nbytes / us / 1e3, 1), "share_of_hbm_peak": round(nbytes / us / 1e-6 / HBM_BYTES_PER_S, 3),
                      "heightfield_bytes_l2": n * HF_BYTES_PER_ENV, "gpu": gpu_info()}))


if __name__ == "__main__":
    main()
