#!/usr/bin/env python
"""Secondary workloads of BASELINE.json (not the headline bench line, which is bench.py / config C4):

  --workload vae    configs[2]: PULSE VAE distillation (encoder + prior + decoder), 8192 envs, horizon 32, im_z_fit.yaml nets,
                    minibatch 16384 (512 envs x 32 steps), 6 mini-epochs of AMPAgent._optimize_kin, frozen PNN teacher in the rollout
  --workload reach  configs[4]: latent-space reach task, frozen PULSE prior + decoder, pulse_z_task.yaml policy
                    (361 -> 2048 -> 1024 -> 512 -> 32, SiLU), PPO update on the latent policy; --envs is per GPU

One step = one full iteration (rollout + update) with synthetic simulator state resident in HBM (physics excluded, as in
bench.py).  Prints one JSON line: env-steps/s, the GEMM FLOPs executed and the tensor-pipe fraction of the update phase.
Timing: CUDA events, L2 flush (256 MiB write) before every timed iteration, >= 3 warm-up iterations.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HORIZON, MINIBATCH, MINI_EPOCHS = 32, 16384, 6


def macs(sizes):
    return sum(a * b for a, b in zip(sizes[:-1], sizes[1:]))


def timed_iterations(iteration, steps, warmup, dev):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(warmup):
        flush.fill_(1)
        iteration(False)
        iteration(False)
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(steps):
        flush.fill_(1)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        iteration(True)
        e.record()
        torch.cuda.synchronize()
        total += s.elapsed_time(e)
    return total / steps


class Graphs:
    def __init__(self, enabled=True):
        self.enabled, self.g = enabled, {}
        self.pool = torch.cuda.graph_pool_handle() if enabled else None

    def run(self, key, fn, *args):
        if not self.enabled:
            return fn(*args)
        g = self.g.get(key)
        if g is None:                # first use: eager; second use: capture (records only) + replay -- nothing executes twice
            self.g[key] = False
            return fn(*args)
        if g is False:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self.pool):
                fn(*args)
            self.g[key] = g
        g.replay()


def bench_vae(a, dev):
    from pulse_b200 import _lib
    from pulse_b200.humanoid_im import HumanoidImCompute
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.vae import PulseVAE, TeacherPNN, pd_targets
    from tools.synth import device_step_inputs, device_tables
    lib = _lib.load()
    n, T = a.envs, HORIZON
    num_mb = T * n // MINIBATCH
    ml = MotionLibB200.from_tables(device_tables(n, dev, seed=100, median_frames=150))
    z = device_step_inputs(ml, n, seed=200)
    comp = HumanoidImCompute(ml)
    vae = PulseVAE(device=dev, horizon=T)                                     # im_z_fit.yaml: task_mlp [1536,1024,512], mlp [3096,2048,1024]
    teacher = TeacherPNN(device=dev, prim_units=(1024, 512), composer_units=(1024, 512), num_prim=3)   # env_im_vae.yaml:56-61 (phc_3 / phc_comp_3)
    obses = torch.zeros(n, T, 934, device=dev)
    obs_carry = torch.zeros(n, 934, device=dev)
    gt_actions = torch.zeros(n, T, 69, device=dev)
    progress_rec = torch.zeros(n, T, dtype=torch.int64, device=dev)
    rewards = torch.zeros(T, n, device=dev)
    values = torch.zeros(T, n, 1, device=dev)
    reward_raw = torch.zeros(n, 5, device=dev)
    reset_buf = torch.zeros(n, dtype=torch.long, device=dev)
    term_buf = torch.zeros(n, dtype=torch.long, device=dev)
    amp_buf = torch.zeros(n, 10, 196, device=dev)
    pd_off, pd_scale, pd_out = torch.zeros(69, device=dev), torch.ones(69, device=dev), torch.zeros(n, 69, device=dev)
    progress0 = z["progress_buf"].clone()
    step_kw = dict(body_state=z["body_state"], dof_vel=z["dof_vel"], dof_force=z["dof_force"], progress_buf=z["progress_buf"],
                   motion_ids=z["motion_ids"], motion_start_times=z["motion_start_times"], motion_start_offset=z["motion_start_offset"],
                   global_offset=z["global_offset"], cycle_counter=z["cycle_counter"], reward_raw=reward_raw, reset_buf=reset_buf,
                   terminate_buf=term_buf)
    comp.step(obs_buf=obs_carry, rew_buf=rewards[0], **step_kw)
    obs_f, gt_f, prog_f = obses.view(T * n, 934), gt_actions.view(T * n, 69), progress_rec.view(T * n)
    graphs = Graphs(os.environ.get("PULSE_NO_GRAPHS", "0") != "1")
    ev = []

    host = {k: z[k].cpu().pin_memory() for k in ("body_state", "dof_state", "dof_force")}
    h_rew = torch.empty(n).pin_memory()
    io = {"on": False, "h2d": sum(v.numel() * 4 for v in host.values()), "d2h": n * 4}

    def rollout_step(t):
        if io["on"]:
            for k, v in host.items():
                z[k].copy_(v, non_blocking=True)
        res = vae.act(obses[:, t])                                            # encoder + decoder + critic_z + critic (K17)
        values[t].copy_(res["values"])
        gt_actions[:, t].copy_(teacher.gt_action(obses[:, t]))                # frozen PNN + composer (K19), HumanoidImDistill.step
        progress_rec[:, t].copy_(z["progress_buf"])                           # kin_dict['progress_buf'] (humanoid_im_distill.py:205)
        pd_targets(res["mus"], pd_off, pd_scale, out=pd_out)                  # env stepped with the mean action (amp_agent.py:244-246), K22
        z["progress_buf"] += 1
        nxt = obses[:, t + 1] if t + 1 < T else obs_carry
        comp.step(obs_buf=nxt, rew_buf=rewards[t], **step_kw)                 # K1-K5
        comp.amp_obs(body_state=z["body_state"], dof_pos=z["dof_pos"], dof_vel=z["dof_vel"], amp_obs_buf=amp_buf)   # K6
        if io["on"]:
            h_rew.copy_(rewards[t], non_blocking=True)

    def update_mb(i):
        r0, r1 = i * MINIBATCH, (i + 1) * MINIBATCH
        vae.optimize_kin(obs_f[r0:r1], gt_f[r0:r1], prog_f[r0:r1], update_obs_rms=True)   # K17 + K18

    def iteration(record):
        z["progress_buf"].copy_(progress0)
        obses[:, 0].copy_(obs_carry)
        for t in range(T):
            graphs.run(("roll", t, io["on"]), rollout_step, t)
        if record:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
        for _ in range(MINI_EPOCHS):
            for i in range(num_mb):
                graphs.run(("upd", i), update_mb, i)
        if record:
            e.record()
            ev.append((s, e))

    en, graphs.enabled = graphs.enabled, False
    iteration(False)
    l0 = lib.pulse_launch_count()
    iteration(False)
    launches = lib.pulse_launch_count() - l0
    graphs.enabled = en
    ms = timed_iterations(iteration, a.steps, a.warmup, dev)
    u_ms = sum(s.elapsed_time(e) for s, e in ev) / len(ev)
    io["on"] = True
    ms_e2e = timed_iterations(iteration, max(2, a.steps // 2), 1, dev)
    io["on"] = False
    enc = macs([960, 1536, 1024, 512, 160, 64])
    pri = macs([384, 1536, 1024, 512, 64])
    dec = macs([448, 3096, 2048, 1024, 69])
    # update: fwd + wgrad for every layer, dgrad for all but the first layer of each net, + the decoder's latent input gradient
    dg = lambda sizes: macs(sizes[1:])
    upd = 3 * (enc + pri + dec) - (960 * 1536 + 384 * 1536 + 448 * 3096) + 3096 * 32
    upd_flops = 2.0 * MINI_EPOCHS * upd * T * n
    critic = macs([960, 1536, 1024, 512, 32]) + macs([448, 3096, 2048, 1024, 1])
    teach = 3 * macs([960, 1024, 512, 69]) + macs([960, 1024, 512, 3])
    roll = enc + dec + critic + teach
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    peak_tf = float(peaks.get("bf16_tflops_sustained", 989.0))   # fallback: H100 SXM data sheet, dense bf16
    L = vae.losses(MINIBATCH)
    return {
        "workload": "PULSE VAE distillation (BASELINE configs[2]): %d envs, horizon 32, im_z_fit.yaml nets, minibatch 16384, 6 mini-epochs" % n,
        "value": T * n / (ms * 1e-3), "unit": "env-steps/s", "ms_per_iteration": ms, "update_ms": u_ms, "rollout_ms": ms - u_ms,
        "e2e": {"value": T * n / (ms_e2e * 1e-3), "unit": "env-steps/s", "h2d_bytes_per_step": T * io["h2d"], "d2h_bytes_per_step": T * io["d2h"],
                "ms_per_step": ms_e2e},
        "gpu_launches": int(launches), "cuda_graphs": graphs.enabled,
        "mflop_per_env_step": 2e-6 * (roll + MINI_EPOCHS * upd),
        "roofline_update": {"bound": "tensor", "achieved": upd_flops / (u_ms * 1e-3) / 1e12, "peak": peak_tf, "unit": "TFLOP/s",
                            "frac": upd_flops / (u_ms * 1e-3) / 1e12 / peak_tf,
                            "note": "algorithmic GEMM FLOPs of the 6 x %d _optimize_kin minibatches / update-phase time (all kernels)" % num_mb},
        "phases": ["32x [obs normalise, encoder + reparam + decoder fwd, critic_z + critic fwd, frozen PNN teacher (3 columns + composer), "
                   "PD targets, fused reward/reset/obs kernel, AMP obs kernel]",
                   "6 x %d minibatches: obs-RMS update, encoder / prior / decoder fwd, action-norm + KL + AR(1) losses, explicit backward, "
                   "grad-norm clip + Adam(5e-4)" % num_mb],
        "not_run": ["discriminator reward over the horizon and GAE (computed by the reference in play_steps but unused by the kin loss)"],
        "last_losses": L, "l2": "256 MiB flush write before every timed iteration", "physics": "excluded",
    }


def bench_reach(a, dev):
    from pulse_b200 import _lib
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.reach import REACH_OBS, ReachTaskB200
    from pulse_b200.rollout import discount_values
    from pulse_b200.vae import PulseVAE, pd_targets
    lib = _lib.load()
    n, T = a.envs, HORIZON
    mb_rows = min(MINIBATCH, T * n)
    num_mb = T * n // mb_rows
    g = torch.Generator(device=dev).manual_seed(3)
    body = torch.zeros(n, 24, 13, device=dev)
    body[..., 0:3] = torch.randn(n, 24, 3, generator=g, device=dev) * 0.3 + torch.tensor([0.0, 0.0, 0.9], device=dev)
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 24, 4, generator=g, device=dev), dim=-1)
    body[..., 7:13] = torch.randn(n, 24, 6, generator=g, device=dev)
    contact = torch.zeros(n, 24, 3, device=dev)
    progress = torch.randint(0, 100, (n,), generator=g, device=dev)
    progress0 = progress.clone()
    task = ReachTaskB200(n, device=dev)
    vae = PulseVAE(device=dev, with_critic=False)                              # frozen prior + decoder of the distilled checkpoint
    policy = PPOPolicy(obs_size=REACH_OBS, num_actions=32, units=(2048, 1024, 512), act="silu", device=dev, seed=0)   # pulse_z_task.yaml:27-28
    obses = torch.zeros(n, T, REACH_OBS, device=dev)
    actions, mus = torch.zeros(n, T, 32, device=dev), torch.zeros(n, T, 32, device=dev)
    neglogp = torch.zeros(n, T, device=dev)
    values, next_values = torch.zeros(T, n, 1, device=dev), torch.zeros(T, n, 1, device=dev)
    rewards, dones = torch.zeros(T, n, device=dev), torch.zeros(T, n, device=dev)
    pd_off, pd_scale, pd_out = torch.zeros(69, device=dev), torch.ones(69, device=dev), torch.zeros(n, 69, device=dev)
    adv_buf, ret_buf = torch.zeros(T * n, device=dev), torch.zeros(T * n, device=dev)
    task.post_physics_step(body, progress)
    obs_f, act_f, mu_f, nlp_f = obses.view(T * n, REACH_OBS), actions.view(T * n, 32), mus.view(T * n, 32), neglogp.view(T * n)
    graphs = Graphs(os.environ.get("PULSE_NO_GRAPHS", "0") != "1")
    ev = []

    host = {"body": body.cpu().pin_memory(), "contact": contact.cpu().pin_memory()}
    h_rew = torch.empty(n).pin_memory()
    io = {"on": False, "h2d": sum(v.numel() * 4 for v in host.values()), "d2h": n * 4}

    def rollout_step(t):
        if io["on"]:
            body.copy_(host["body"], non_blocking=True)
            contact.copy_(host["contact"], non_blocking=True)
        obses[:, t].copy_(task.obs_buf)
        res = policy.act(obses[:, t])                                          # latent policy (K20 caller)
        actions[:, t].copy_(res["actions"]); mus[:, t].copy_(res["mus"]); neglogp[:, t].copy_(res["neglogpacs"]); values[t].copy_(res["values"])
        dec = vae.compute_z_actions(task.obs_buf, res["actions"])             # HumanoidZ.compute_z_actions: prior + decoder (K20)
        pd_targets(dec, pd_off, pd_scale, out=pd_out)                         # pre_physics_step (K22)
        task.update_task(progress)                                            # _update_task
        progress.add_(1)                                                      # physics would run here (excluded)
        task.post_physics_step(body, progress, contact)                       # reward + reset + obs (K21)
        rewards[t].copy_(task.rew_buf); dones[t].copy_(task.reset_buf)
        nv = policy.critic_values(task.obs_buf)
        next_values[t].copy_(nv * (1.0 - task._terminate_buf.unsqueeze(1).float()))
        if io["on"]:
            h_rew.copy_(rewards[t], non_blocking=True)

    def post_rollout():
        adv, ret = discount_values(dones, values, rewards.unsqueeze(-1), next_values, normalize_advantage=True)
        policy.value_rms.update(values.view(T * n, 1))
        adv_buf.copy_(adv)
        ret_buf.copy_(policy.value_rms.normalize_values(ret.view(-1, 1)).view(-1))   # statistics include the values batch, not yet the returns
        policy.value_rms.update(ret.view(-1, 1))

    def update_mb(i):
        r0, r1 = i * mb_rows, (i + 1) * mb_rows
        policy.train_minibatch(obs_f[r0:r1], act_f[r0:r1], nlp_f[r0:r1], adv_buf[r0:r1], ret_buf[r0:r1], old_mu=mu_f[r0:r1])

    def iteration(record):
        progress.copy_(progress0)
        for t in range(T):
            graphs.run(("roll", t, io["on"]), rollout_step, t)
        graphs.run(("post",), post_rollout)
        if record:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
        for _ in range(MINI_EPOCHS):
            for i in range(num_mb):
                graphs.run(("upd", i), update_mb, i)
        if record:
            e.record()
            ev.append((s, e))

    en, graphs.enabled = graphs.enabled, False
    iteration(False)
    l0 = lib.pulse_launch_count()
    iteration(False)
    launches = lib.pulse_launch_count() - l0
    graphs.enabled = en
    ms = timed_iterations(iteration, a.steps, a.warmup, dev)
    u_ms = sum(s.elapsed_time(e) for s, e in ev) / len(ev)
    io["on"] = True
    ms_e2e = timed_iterations(iteration, max(2, a.steps // 2), 1, dev)
    io["on"] = False
    pol = macs([384, 2048, 1024, 512, 32])
    crit = macs([384, 2048, 1024, 512, 1])
    zdec = macs([384, 1536, 1024, 512, 64]) + macs([448, 3096, 2048, 1024, 69])
    upd = 3 * (pol + crit) - 2 * 384 * 2048
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    peak_tf = float(peaks.get("bf16_tflops_sustained", 989.0))   # fallback: H100 SXM data sheet, dense bf16
    upd_flops = 2.0 * MINI_EPOCHS * upd * T * n
    return {
        "workload": "latent-space reach task (BASELINE configs[4]): %d envs on this GPU, frozen PULSE prior + decoder, pulse_z_task.yaml policy" % n,
        "value": T * n / (ms * 1e-3), "unit": "env-steps/s", "ms_per_iteration": ms, "update_ms": u_ms, "rollout_ms": ms - u_ms,
        "e2e": {"value": T * n / (ms_e2e * 1e-3), "unit": "env-steps/s", "h2d_bytes_per_step": T * io["h2d"], "d2h_bytes_per_step": T * io["d2h"],
                "ms_per_step": ms_e2e},
        "gpu_launches": int(launches), "cuda_graphs": graphs.enabled, "mflop_per_env_step": 2e-6 * (pol + 2 * crit + zdec + MINI_EPOCHS * upd),
        "roofline_update": {"bound": "tensor", "achieved": upd_flops / (u_ms * 1e-3) / 1e12, "peak": peak_tf, "unit": "TFLOP/s",
                            "frac": upd_flops / (u_ms * 1e-3) / 1e12 / peak_tf},
        "phases": ["32x [latent policy + critic fwd, Gaussian sample, prior + decoder decode (K20), PD targets (K22), target resample, "
                   "reach reward/reset/obs kernel (K21), critic fwd on next obs]", "GAE + returns + adv-norm",
                   "6 x %d minibatches of %d rows: PPO losses, backward, clip + Adam" % (num_mb, mb_rows)],
        "l2": "256 MiB flush write before every timed iteration", "physics": "excluded",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["vae", "reach"], required=True)
    ap.add_argument("--envs", type=int, default=None)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    if a.envs is None:
        a.envs = 8192 if a.workload == "vae" else 1024     # reach: 8192 envs over 8 GPUs
    out = bench_vae(a, dev) if a.workload == "vae" else bench_reach(a, dev)
    out.update(steps=a.steps, warmup=a.warmup, data="synthetic", dtype="bf16 GEMM operands, fp32 accumulate / master weights")
    s = json.dumps(out)
    print(s, flush=True)
    if a.json:
        open(a.json, "w").write(s + "\n")


if __name__ == "__main__":
    main()
