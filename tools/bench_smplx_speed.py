#!/usr/bin/env python
"""The PULSE-X speed task on the device (HumanoidSpeedZ, robot=smplx_humanoid, env_pulsex_amp.yaml): full training iterations of the
52-body SMPL-X humanoid through `ZTaskStepsB200`, measured as tools/bench_ztask_rollout.py measures the SMPL latent tasks, and the step
kernel alone.  --task reach / strike measures the PULSE-X reach or strike task the same way (HumanoidReachZ / HumanoidStrikeZ, reach
body R_Wrist 36, strike bodies R_Elbow, R_Wrist and the right index finger's base 35, 36, 37), and times `pulse_smplx_target_step`
alternated sample by sample with `pulse_smplx_speed_step` in the same call, so the two rates compare.

  iteration  one horizon (device resets inside it, latent policy 2048-1024-512 SiLU over 48 latent dimensions, frozen prior + 778 -> 153
             decoder of the PULSE-X VAE's shapes with random weights, pre-physics and step kernels; no physics), then `finish` and the
             PPO update (6 mini-epochs of 16384-row minibatches), on synthetic 52-body MotionLib tables and simulator state.  Two arms
             alternated iteration by iteration: graph (as shipped) and eager (use_graphs=False).  Milliseconds per horizon and update
             from device events after --warmup, with an L2 flush before each timed region, over --iters iterations.  --policy direct
             measures the PPO baseline instead (HumanoidSpeed / HumanoidReach / HumanoidStrike under learning=ppo: ZTaskStepsB200 with
             vae=None, the same network acting in the 153 dofs, no prior or decoder); --policy both alternates the latent and the direct
             drivers' arms iteration by iteration, on MotionLib tables and simulator state built from the same seeds.
  step       `pulse_smplx_speed_step` alone at --step-envs envs: device events around --step-reps back-to-back launches (one L2
             flush before each sample), beside the bytes one env-step reads and writes as computed from the shapes (52 x 13 body
             floats, 52 x 3 contact floats, the 781-float observation row, and the per-env scalars).  At 16384 envs a launch touches
             ~106 MB, more than the 50 MB L2, so the back-to-back launches stream mostly from HBM.

One JSON line per measurement, with the card name, power limit and maximum SM clock read in the same call.  Needs a CUDA device.

  python tools/bench_smplx_speed.py [--task speed|reach|strike] [--policy latent|direct|both] [--envs 1536 8192] [--iters 5] [--warmup 2] [--step-envs 16384] [--step-reps 200]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_ztask_rollout import HORIZON, MINI_EPOCHS, MINIBATCH, POLICIES, UNITS, gpu_info   # noqa: E402

B, D, LATENT = 52, 153, 48
CONTACT_IDS = (7, 3, 8, 4)          # R_Ankle, L_Ankle, R_Toe, L_Toe in the SMPLH_MUJOCO_NAMES order


def tables(clips, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    nf = torch.randint(60, 240, (clips,), device=dev, generator=g)
    F = int(nf.sum())
    unit = lambda q: q / q.norm(dim=-1, keepdim=True)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    dt = torch.full((clips,), 1.0 / 30.0, device=dev)
    return dict(gts=r(F, B, 3) * 0.3 + torch.tensor([0.0, 0.0, 0.9], device=dev), grs=unit(r(F, B, 4)), lrs=unit(r(F, B, 4)), gvs=r(F, B, 3),
                gavs=r(F, B, 3), dvs=r(F, B - 1, 3), lengths=dt * (nf - 1).float(), num_frames=nf, dt=dt,
                length_starts=torch.cumsum(nf, 0) - nf)


def sim_state(n, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    body = torch.zeros(n, B + 1, 13, device=dev)
    body[..., 0:3] = torch.randn(n, B + 1, 3, device=dev, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9], device=dev)
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, B + 1, 4, device=dev, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, B + 1, 6, device=dev, generator=g)
    contact = torch.zeros(n, B + 1, 3, device=dev)
    body[::16, 40, 2], contact[::16, 40, 2] = 0.05, 5.0                                     # fallen: reset at the second step
    dof_state = torch.randn(n, D, 2, device=dev, generator=g)
    return dict(body_state=body, root_states=body[:, 0].clone(), dof_pos=dof_state[:, :, 0], dof_vel=dof_state[:, :, 1], contact_forces=contact,
                progress_buf=torch.randint(2, 300, (n,), device=dev, generator=g), sampled_motion_ids=torch.zeros(n, dtype=torch.int64, device=dev),
                motion_start_times=torch.zeros(n, device=dev))


REACH_BODY, STRIKE_IDS = 36, (35, 36, 37)


def make_task(kind, n, dev):
    from pulse_b200.ztasks import SmplxReachTaskB200, SmplxSpeedTaskB200, SmplxStrikeTaskB200
    if kind == "reach":
        return SmplxReachTaskB200(n, device=dev, reach_body_id=REACH_BODY, contact_body_ids=CONTACT_IDS)
    if kind == "strike":
        return SmplxStrikeTaskB200(n, device=dev, strike_body_ids=STRIKE_IDS, contact_body_ids=CONTACT_IDS)
    return SmplxSpeedTaskB200(n, device=dev, contact_body_ids=CONTACT_IDS)


def with_target(s, n, dev):
    """The strike task's target views: body 53 of an [N, 54, 13] rigid-body tensor's contact rows and an [N, 2, 13] actor root tensor."""
    g = torch.Generator(device=dev).manual_seed(400)
    roots = torch.randn(n, 2, 13, device=dev, generator=g)
    roots[:, 1, 3:7] = torch.nn.functional.normalize(roots[:, 1, 3:7], dim=-1)
    s["target_states"], s["tar_contact_forces"] = roots[:, 1], s["contact_forces"][:, B]
    return s


def build(n, dev, use_graphs, kind="speed", policy="latent"):
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.vae import PulseVAE
    from pulse_b200.ztask_reset import SmplxTargetResetB200, ZTaskResetB200
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    ml = MotionLibB200.from_tables(tables(256, dev, 100))
    g = torch.Generator(device=dev).manual_seed(300)
    floor = -0.9 + 0.05 * torch.rand(ml.gts.shape[0], device=dev, generator=g)            # stand-in for the ground table
    task = make_task(kind, n, dev)
    if policy == "direct":                                                                  # ppo.yaml: the policy writes the 153 dof targets
        pol, vae = PPOPolicy(obs_size=task.obs_size, num_actions=D, units=UNITS, act="silu", logstd=-2.9, device=dev, seed=0), None
    else:
        pol = PPOPolicy(obs_size=task.obs_size, num_actions=LATENT, units=UNITS, act="silu", device=dev, seed=0)
        vae = PulseVAE(self_obs_size=778, num_actions=D, latent=LATENT, device=dev, with_critic=False)
    reset = ZTaskResetB200("speed", ml, floor, upright=False) if kind == "speed" else SmplxTargetResetB200(kind, ml, floor, upright=False)
    sim = sim_state(n, dev, 200)
    if kind == "strike":
        sim = with_target(sim, n, dev)
    drv = ZTaskStepsB200(task, reset, pol, vae, sim, horizon=HORIZON, use_graphs=use_graphs, reset_seed=1)
    drv.first_observation()
    return drv


def step_bytes(kind="speed"):
    """Bytes one env-step of pulse_smplx_speed_step moves, from the shapes: reads the 52 x 13 body floats, 52 x 3 contact floats, the
    52 termination heights (cached across envs: not counted), progress, prev_root_pos and tar_speed; writes the 781-float observation
    row, reward, reward_raw, reset and terminate.  Reach reads tar_pos instead of prev_root_pos / tar_speed and writes no reward_raw;
    strike reads prev_root_pos, the 13-float target state and its 3-float contact force, and writes a 793-float row."""
    rd = {"body_state": B * 13 * 4, "contact_forces": B * 3 * 4, "progress/prev_root/tar_speed": 8 + 12 + 4}
    wr = {"obs_row": 781 * 4, "rew/reward_raw": 8, "reset/terminate": 16}
    if kind == "reach":
        rd, wr = dict(rd), dict(wr)
        del rd["progress/prev_root/tar_speed"], wr["rew/reward_raw"]
        rd["progress/tar_pos"], wr["rew"] = 8 + 12, 4
    elif kind == "strike":
        rd = {"body_state": B * 13 * 4, "contact_forces": B * 3 * 4, "progress/prev_root": 8 + 12, "target_state": 13 * 4, "tar_contact": 3 * 4}
        wr = {"obs_row": 793 * 4, "rew": 4, "reset/terminate": 16}
    return rd, wr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", choices=("speed", "reach", "strike"), default="speed")
    ap.add_argument("--policy", choices=tuple(POLICIES), default="latent")
    ap.add_argument("--envs", type=int, nargs="+", default=[1536, 8192])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--step-envs", type=int, default=16384)
    ap.add_argument("--step-reps", type=int, default=200)
    args = ap.parse_args()
    if args.iters < 3:
        raise SystemExit("at least three timed iterations")
    if not torch.cuda.is_available():
        raise SystemExit("bench_smplx_speed.py needs a CUDA device")
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
        arms = {(pol, mode): build(n, dev, mode == "graph", args.task, pol) for pol in pols for mode in ("graph", "eager")}
        mb = min(MINIBATCH, n * HORIZON)
        update = lambda d: (d.finish(), d.train_epoch(mini_epochs=MINI_EPOCHS, minibatch=mb))
        ev = {a: {"horizon": [], "update": []} for a in arms}
        resets = {a: 0.0 for a in arms}
        for it in range(args.warmup + args.iters):
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
            what = ("PULSE-X %s task iteration (Humanoid%sZ, smplx_humanoid, 52 bodies, 153 dofs): %d envs, horizon %d, latent policy %s SiLU "
                    "over %d dims, frozen prior + 778->153 decoder" if pol == "latent" else
                    "PPO baseline %s task iteration (Humanoid%s, smplx_humanoid, 52 bodies, ppo.yaml): %d envs, horizon %d, policy %s SiLU "
                    "over the %d dofs, no prior or decoder")
            out = {"workload": (what + ", task reward only, %d mini-epochs of %d rows, no physics")
                               % (args.task, args.task.capitalize(), n, HORIZON, "-".join(map(str, UNITS)), LATENT if pol == "latent" else D,
                                  MINI_EPOCHS, mb),
                   "gpu": info, "envs": n, "iters": args.iters, "warmup": args.warmup, "policy": pol,
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

    # the step kernel alone; with --task reach / strike the target step and the speed step, alternated sample by sample
    n = args.step_envs
    kinds = ["speed"] if args.task == "speed" else [args.task, "speed"]
    s = sim_state(n, dev, 7)
    if args.task == "strike":
        s = with_target(s, n, dev)
    st = _lib.current_stream(dev)
    calls = {}
    for kind in kinds:
        task = make_task(kind, n, dev)
        a = task._args(s["body_state"], s["progress_buf"], s["contact_forces"])
        if kind == "strike":
            a.target_states, a.target_env_stride = s["target_states"].data_ptr(), s["target_states"].stride(0)
            a.tar_contact_forces, a.tar_contact_env_stride = s["tar_contact_forces"].data_ptr(), s["tar_contact_forces"].stride(0)
        fn = "pulse_smplx_speed_step" if kind == "speed" else "pulse_smplx_target_step"
        calls[kind] = (fn, getattr(lib, fn), a, task)
    for fn, f, a, _ in calls.values():
        for _ in range(10):
            _lib.check(f(C.byref(a), n, st), fn)
    times = {k: [] for k in kinds}
    for _ in range(5):
        for kind in kinds:
            fn, f, a, _ = calls[kind]
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.step_reps):
                _lib.check(f(C.byref(a), n, st), fn)
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1) * 1e3 / args.step_reps)
    for kind in kinds:
        rd, wr = step_bytes(kind)
        per_env = sum(rd.values()) + sum(wr.values())
        us = sorted(times[kind])[len(times[kind]) // 2]
        name = calls[kind][0] + ("" if kind == "speed" else " (%s)" % kind)
        print(json.dumps({"workload": "%s alone: %d envs, %d back-to-back launches per sample, median of 5 samples" % (name, n, args.step_reps),
                          "gpu": info, "envs": n, "kernel_us": round(us, 2), "kernel_us_samples": [round(t, 2) for t in times[kind]],
                          "bytes_per_env_step": {"read": rd, "write": wr, "total": per_env},
                          "achieved_GB_per_s": round(per_env * n / (us * 1e-6) / 1e9, 1)}), flush=True)


if __name__ == "__main__":
    main()
