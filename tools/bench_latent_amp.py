"""Times the latent-space tasks' training iteration with and without the discriminator, and the AMP buffers' own work.

Per task and env count one JSON line: the card's name, power limit and maximum SM clock (read in the same call); for each of the four
arms (no discriminator / discriminator x graph / eager) the horizon (play_steps) and update (finish + train_epoch) times as CUDA-event
means with min / max over the timed iterations; with the discriminator the per-epoch AMP work timed alone on the graph arm's buffers
(a demo fetch of amp_batch_size rows, the demo and replay samples of n*T rows, the replay store of n*T rows) and the one-time fill of the
demo ring.  The drivers are the ones tools/bench_ztask_rollout.py, bench_terrain_rollout.py and bench_imz_rollout.py build (synthetic
MotionLib and simulator state, no physics); the discriminator arm swaps in the same policy with the discriminator of the configs
(1024-512 ReLU, disc_coef 5) and an AmpBuffersB200 of the learning configs' sizes (200 000-row rings, amp_batch_size 512,
amp_minibatch_size 4096, keep probability 0.01), disc_reward_w 0.

The smplx-speed task is the PULSE-X speed driver of tools/bench_smplx_speed.py (52 bodies, 48 latent dimensions) with 10 x 465-float
AMP rows (env_pulsex_amp.yaml) and a 4650-wide discriminator input; for it a last line times `pulse_smplx_amp_obs_row` alone at
--row-envs envs (device events around --row-reps back-to-back launches, median of 5 samples, one L2 flush before each) beside the bytes
one env-step moves as computed from the shapes.

  python tools/bench_latent_amp.py --task speed --envs 1536 8192
  python tools/bench_latent_amp.py --task vr --envs 3072
  python tools/bench_latent_amp.py --task smplx-speed --envs 1536 8192
"""
import ctypes as C
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import bench_imz_rollout as bimz          # noqa: E402
from tools import bench_smplx_speed as bsx           # noqa: E402
from tools import bench_terrain_rollout as bter      # noqa: E402
from tools import bench_ztask_rollout as bzt         # noqa: E402

HORIZON, MINIBATCH, MINI_EPOCHS = 32, 16384, 6


def build(task, n, dev, use_graphs, disc, terrain=None):
    """The benchmark driver of `task`; with `disc`, rebuilt on the same pieces with the discriminator and the AMP part."""
    from pulse_b200.amp_buffers import AmpBuffersB200
    from pulse_b200.imz_rollout import ImZStepsB200
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.sept import SeptPolicy
    from pulse_b200.terrain_rollout import TerrainStepsB200
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    if task == "terrain":
        d0 = bter.build(n, dev, use_graphs, *terrain)
    elif task == "vr":
        d0 = bimz.build(n, dev, use_graphs)
    elif task == "smplx-speed":
        d0 = bsx.build(n, dev, use_graphs)
    else:
        d0 = bzt.build(task, n, dev, use_graphs)
    if not disc:
        return d0
    kw = dict(horizon=HORIZON, use_graphs=use_graphs, reset_seed=1)
    if task == "vr":
        amp = AmpBuffersB200(d0.comp.motion_lib, amp_width=196, upright=True)
        pol = PPOPolicy(obs_size=d0.comp.obs_size, num_actions=32, units=bimz.UNITS, act="silu", logstd=-1.5, device=dev, seed=0,
                        with_disc=True, amp_obs_size=amp.row_floats)
        d = ImZStepsB200(d0.comp, pol, d0.vae, d0.sim, amp=amp, **kw)
    else:
        amp = AmpBuffersB200(d0.reset.motion_lib, amp_width=d0.reset.amp_width, upright=d0.reset.upright)
        if task == "terrain":
            pol = SeptPolicy(num_actions=32, with_disc=True, amp_obs_size=amp.row_floats, device=dev, seed=0)
            d = TerrainStepsB200(d0.task, d0.reset, pol, d0.vae, d0.sim, amp=amp, **kw)
        else:
            pol = PPOPolicy(obs_size=d0.task.obs_size, num_actions=bsx.LATENT if task == "smplx-speed" else 32, units=bzt.UNITS, act="silu",
                            device=dev, seed=0, with_disc=True, amp_obs_size=amp.row_floats)
            d = ZTaskStepsB200(d0.task, d0.reset, pol, d0.vae, d0.sim, amp=amp, **kw)
    d.first_observation()
    return d


def row_bytes(width=465, steps=10):
    """Bytes one env-step of pulse_smplx_amp_obs_row moves, from the shapes: reads the (steps - 1) history rows, the root's 13 body floats,
    the 4 key bodies' positions and the 49 kept joints' 147 dof positions and velocities; writes the steps x width row."""
    rd = {"history": (steps - 1) * width * 4, "state": (13 + 4 * 3 + 2 * 147) * 4}
    wr = {"row": steps * width * 4}
    return rd, wr


def time_row(n, reps, dev, flush):
    """pulse_smplx_amp_obs_row alone: microseconds per launch (median of 5 samples of `reps` launches) and the shapes' bytes."""
    from pulse_b200 import _lib
    lib = _lib.load()
    s = bsx.sim_state(n, dev, 7)
    W = 465
    prev, out = torch.randn(n, 10 * W, device=dev), torch.zeros(n, 10 * W, device=dev)
    a = _lib.AmpRowArgs(body_state=s["body_state"].data_ptr(), body_env_stride=s["body_state"].stride(0), dof_pos=s["dof_pos"].data_ptr(),
                        dof_vel=s["dof_vel"].data_ptr(), dof_env_stride=s["dof_pos"].stride(0), dof_elem_stride=s["dof_pos"].stride(1),
                        prev=prev.data_ptr(), ld_prev=10 * W, out=out.data_ptr(), ld_out=10 * W, num_steps=10, amp_width=W, remove_base_rot=1)
    st = _lib.current_stream(dev)
    for _ in range(10):
        _lib.check(lib.pulse_smplx_amp_obs_row(C.byref(a), n, st), "pulse_smplx_amp_obs_row")
    times = []
    for _ in range(5):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            _lib.check(lib.pulse_smplx_amp_obs_row(C.byref(a), n, st), "pulse_smplx_amp_obs_row")
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / reps)
    rd, wr = row_bytes(W)
    per_env = sum(rd.values()) + sum(wr.values())
    us = sorted(times)[len(times) // 2]
    return {"workload": "pulse_smplx_amp_obs_row alone: %d envs, 10 x %d floats, %d back-to-back launches per sample, median of 5 samples"
                        % (n, W, reps), "envs": n, "kernel_us": round(us, 2), "kernel_us_samples": [round(t, 2) for t in times],
            "bytes_per_env_step": {"read": rd, "write": wr, "total": per_env}, "MB_per_launch": round(per_env * n / 1e6, 1),
            "achieved_GB_per_s": round(per_env * n / (us * 1e-6) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", choices=("reach", "speed", "strike", "terrain", "vr", "smplx-speed"), default="speed")
    ap.add_argument("--envs", type=int, nargs="+", default=[1536, 8192])
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--amp-reps", type=int, default=10)
    ap.add_argument("--row-envs", type=int, default=16384)
    ap.add_argument("--row-reps", type=int, default=200)
    args = ap.parse_args()
    if args.iters < 3:
        raise SystemExit("at least three timed iterations")
    if not torch.cuda.is_available():
        raise SystemExit("bench_latent_amp.py needs a CUDA device")
    dev = "cuda:0"
    info = bzt.gpu_info()
    terrain = bter.terrain_tables(dev) if args.task == "terrain" else None
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)                  # larger than the 50 MB L2

    def timed(fn):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        return s, e

    def ms(pairs):
        torch.cuda.synchronize()
        v = [s.elapsed_time(e) for s, e in pairs]
        return {"mean": round(sum(v) / len(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}

    for n in args.envs:
        mb = min(MINIBATCH, n * HORIZON)
        out = {"workload": "latent-space %s task iteration: %d envs, horizon %d, %d mini-epochs of %d rows, no physics; the discriminator "
                           "arms train it (disc_reward_w 0) with 200 000-row demo and replay rings" % (args.task, n, HORIZON, MINI_EPOCHS, mb),
               "gpu": info, "task": args.task, "envs": n, "iters": args.iters, "warmup": args.warmup}
        for disc in (False, True):
            arms = {}
            for mode in ("graph", "eager"):
                torch.cuda.empty_cache()
                d = build(args.task, n, dev, mode == "graph", disc, terrain)
                if disc:
                    fill = timed(d.amp.init_demo)
                    out["demo_ring_fill_ms"] = ms([fill])["mean"]
                ev = {"horizon": [], "update": []}
                for it in range(args.warmup + args.iters):
                    h = timed(d.play_steps)
                    u = timed(lambda: (d.finish(), d.train_epoch(mini_epochs=MINI_EPOCHS, minibatch=mb)))
                    if it >= args.warmup:
                        ev["horizon"].append(h)
                        ev["update"].append(u)
                arms[mode] = {k: ms(v) for k, v in ev.items()}
                if disc and mode == "graph":
                    amp, rows = d.amp, n * HORIZON
                    take, (demo, replay) = d._amp_batches(mb)
                    flat = d.amp_obs.view(rows, -1)
                    parts = {"demo_fetch": lambda: amp.update_demos(), "demo_sample": lambda: amp.sample(amp.demo, rows, mb, demo),
                             "replay_sample": lambda: amp.sample(amp.replay, rows, mb, replay, fallback=flat),
                             "replay_store": lambda: amp.store_replay(flat)}
                    out["amp_epoch_ms"] = {k: ms([timed(f) for _ in range(args.amp_reps)]) for k, f in parts.items()}
                del d
            out["disc" if disc else "no_disc"] = arms
        print(json.dumps(out), flush=True)
    if args.task == "smplx-speed":
        torch.cuda.empty_cache()
        print(json.dumps(dict(time_row(args.row_envs, args.row_reps, dev, flush), gpu=info)), flush=True)


if __name__ == "__main__":
    main()
