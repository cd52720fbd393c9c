"""Speed of the amp_sept policy (pedestrian terrain task, pulse_z_terrain.yaml widths) at a 16384-row minibatch:

  * one SeptPolicy.train_minibatch with the AMP discriminator on 3 x 4096 rows (normalise, task encoder, actor, critic, PPO loss,
    backward incl. the shared encoder, discriminator with its gradient penalty, norm clip + Adam), timed over a CUDA graph of many;
  * act() (normalise, task encoder, actor, critic, sampling);
  * pulse_normalize_split alone (training mode, with the fp64 moments).

  python tools/bench_sept.py [--rows 16384] [--amp-rows 4096] [--steps 20] [--reps 5]

Prints one JSON line: milliseconds, algorithmic TFLOP/s (GEMM multiply-adds x 2, from the layer shapes below) and the split kernel's
algorithmic GB/s, with the card name, power limit and maximum SM clock read in the same run.  Needs a CUDA device: there is no fallback.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

S, TRAJ, HEIGHTS, A, AMP = 358, 20, 1024, 32, 1960
TASK_UNITS, UNITS, DISC_UNITS = (512, 256), (2048, 1024, 512), (1024, 512)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception:
        return "unknown"


def chain(n_in, units, head=None):
    """(K, N) of each Linear of an MLP"""
    dims, k = [], n_in
    for u in list(units) + ([head] if head else []):
        dims.append((k, u))
        k = u
    return dims


def flops(M, B):
    """Algorithmic FLOPs (2 x multiply-adds of the GEMMs) of act() and of one training minibatch."""
    E = TASK_UNITS[-1]
    task = chain(TRAJ + HEIGHTS, TASK_UNITS)
    actor, critic = chain(S + E, UNITS, A), chain(S + E, UNITS, 1)
    disc = chain(AMP, DISC_UNITS, 1)
    mk = lambda dims: sum(k * n for k, n in dims)
    fwd = 2 * M * (mk(task) + mk(actor) + mk(critic))
    # backward: every weight gradient; input gradients of every layer but the first, plus the embedding columns of the first layers
    bwd = 2 * M * (mk(task) + mk(actor) + mk(critic)) + 2 * M * (mk(task[1:]) + mk(actor[1:]) + mk(critic[1:]) + 2 * UNITS[0] * E)
    d_fwd_bwd = 2 * 3 * B * mk(disc) * 2 + 2 * 3 * B * mk(disc[1:])
    (k1, n1), (k2, n2) = disc[0], disc[1]
    penalty = 2 * B * (n2 * n1 + n1 * k1 + n1 * k1 + k1 * n1 + n2 * n1 + n1 * n2)   # the six GEMMs of the analytic gradient penalty (amp.py)
    return fwd, fwd + bwd + d_fwd_bwd + penalty


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16384)
    ap.add_argument("--amp-rows", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sept.py needs a CUDA device")
    from pulse_b200.sept import SeptPolicy
    dev, M, B = "cuda:0", args.rows, args.amp_rows
    torch.manual_seed(0)
    pol = SeptPolicy(self_obs_size=S, task_obs_size_detail={"traj": TRAJ, "heightmap": HEIGHTS}, task_units=TASK_UNITS, units=UNITS,
                     num_actions=A, with_disc=True, amp_obs_size=AMP, disc_units=DISC_UNITS, device=dev)
    g = torch.Generator(device=dev).manual_seed(1)
    obs = torch.randn(M, S + TRAJ + HEIGHTS, device=dev, generator=g)
    amp = tuple(torch.randn(B, AMP, device=dev, generator=g) for _ in range(3))
    out = pol.act(obs)
    actions, nlp, mus = out["actions"].clone(), out["neglogpacs"].clone(), out["mus"].clone()
    adv, ret = torch.randn(M, device=dev, generator=g), torch.randn(M, device=dev, generator=g)
    step = lambda: pol.train_minibatch(obs, actions, nlp, adv, ret, old_mu=mus, amp=amp)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(args.steps):
            step()
    train_ms = [t / args.steps for t in timed(graph.replay, args.reps)]
    act_ms = timed(lambda: [pol.act(obs) for _ in range(args.steps)], args.reps)
    act_ms = [t / args.steps for t in act_ms]
    b = pol._buf(M, True)
    split = lambda: [pol.obs_rms.normalize_split(obs, S, b["x2"][0], TASK_UNITS[-1], b["t2"][0], True) for _ in range(args.steps)]
    split_ms = [t / args.steps for t in timed(split, args.reps)]   # includes the small merge launch of the statistics
    f_act, f_train = flops(M, B)
    p_w, t_w = pol.actor.Kp0 - TASK_UNITS[-1], pol.task.Kp0
    split_bytes = M * (S + TRAJ + HEIGHTS) * 4 + M * (p_w + t_w) * 2   # read the fp32 rows once, write both bf16 operands (not the embedding)
    r = lambda x: round(x, 3)
    print(json.dumps({"rows": M, "amp_rows": B, "train_minibatch_ms": r(min(train_ms)), "train_minibatch_ms_all": [r(t) for t in train_ms],
                      "train_TFLOPs": r(f_train / min(train_ms) / 1e9), "train_GFLOP": r(f_train / 1e9),
                      "act_ms": r(min(act_ms)), "act_ms_all": [r(t) for t in act_ms], "act_TFLOPs": r(f_act / min(act_ms) / 1e9),
                      "split_ms": r(min(split_ms)), "split_ms_all": [r(t) for t in split_ms], "split_MB": r(split_bytes / 1e6),
                      "split_GBps": round(split_bytes / min(split_ms) / 1e6, 1), "gpu": gpu_info()}))


if __name__ == "__main__":
    main()
