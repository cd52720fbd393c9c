"""Evaluation over all clips of a MotionLib with the metrics on the device (SURVEY 8f-2).

Host-side mirror of `IMAmpAgent.eval` / `_post_step_eval` (phc/learning/im_amp.py:136-363) and of
`update_training_data` (:126-132), GPU-first:

  * the reference copies every env's 24 body positions (simulated and reference) to the host EVERY evaluation step
    (`extras['body_pos'] = body_pos.cpu().numpy()`, humanoid_im.py:664-673), keeps Python lists of frames and runs
    `smpl_sim`'s `compute_metrics_lite` over them at the end.  Here one `pulse_eval_step` call per step accumulates the per-frame
    metrics (global / root-relative / Procrustes-aligned MPJPE, velocity and acceleration errors) into per-env fp64 sums, keeps the
    termination state and applies the reference's `curr_max` stopping rule on the device; the host polls ONE flag every
    `poll_every` steps and reads 5 sums + 3 counts per env once per chunk.
  * success rate, failed / success keys and the PMCP sampling-weight update (`MotionDatasetB200.update_*_sampling_weight`) follow
    the reference's bookkeeping exactly (first `num_unique` sequences, chunks of `num_envs`).

`EvalMetricsB200` is the device state of one chunk; `EvalLoopB200` drives chunks through caller-supplied callbacks (reset, step,
load chunk), so it runs in front of Isaac Gym, of the stand-in task of the tests, or of a synthetic simulator.
"""
import ctypes as C
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib

METRIC_NAMES = ("mpjpe_g", "mpjpe_l", "mpjpe_pa", "vel_dist", "accel_dist")     # sums[:, k]; counts columns: 0, 0, 0, 1, 2
_COUNT_COL = (0, 0, 0, 1, 2)


class EvalMetricsB200:
    """Device-side accumulators of one evaluation chunk (num_envs sequences)."""

    def __init__(self, num_envs: int, device="cuda:0", num_bodies: int = 24):
        if num_bodies != 24:
            raise _lib.PulseError("pulse_eval_step is built for the 24-body SMPL humanoid")
        self.N, self.device = int(num_envs), torch.device(device)
        dev = self.device
        self.ctrl = torch.zeros(8, dtype=torch.int32, device=dev)              # step, finished, scratch x3
        self.terminate_state = torch.zeros(self.N, dtype=torch.int32, device=dev)
        self.hist = torch.zeros(self.N, 2, num_bodies, 3, device=dev)
        self.sums = torch.zeros(self.N, 5, dtype=torch.float64, device=dev)
        self.counts = torch.zeros(self.N, 3, dtype=torch.int32, device=dev)
        self.mpjpe = torch.zeros(self.N, device=dev)                            # extras['mpjpe'] of the last step
        self.num_steps = torch.zeros(self.N, dtype=torch.int32, device=dev)
        self.bound, self.max_steps = self.N, 0
        self.lib = _lib.load()

    def begin_chunk(self, num_steps: Sequence[int], bound: Optional[int] = None) -> None:
        """`num_steps` = `_motion_lib.get_motion_num_steps()` of the loaded chunk (motion_lib_base.py:428-432); `bound`: envs
        [0, bound) hold distinct clips -- smaller than num_envs only in the wrapped last chunk (im_amp.py:254-262)."""
        ns = torch.as_tensor(np.asarray(num_steps), dtype=torch.int32)
        if ns.shape[0] != self.N:
            raise _lib.PulseError(f"num_steps has {ns.shape[0]} entries for {self.N} envs")
        self.num_steps.copy_(ns)
        self.max_steps = int(ns.max())
        self.bound = self.N if bound is None else int(bound)
        for t in (self.ctrl, self.terminate_state, self.hist, self.sums, self.counts):
            t.zero_()

    def step(self, body_pos: torch.Tensor, body_pos_gt: torch.Tensor, terminate: torch.Tensor) -> None:
        """One evaluation step: body_pos = the simulator's rigid-body positions ([N, B>=24, >=3] view, e.g. `_rigid_body_state`),
        body_pos_gt = `motion_res['rg_pos']` [N, 24, 3], terminate = `terminate_buf` (int64 [N]).  No host synchronisation."""
        for name, t in (("body_pos", body_pos), ("body_pos_gt", body_pos_gt)):
            if t.dim() != 3 or t.shape[0] != self.N or t.shape[1] < 24 or t.stride(2) != 1 or t.dtype != torch.float32:
                raise _lib.PulseError(f"{name}: expected a float32 [N, >=24, >=3] view with unit inner stride")
        if terminate.dtype != torch.int64 or not terminate.is_contiguous():
            raise _lib.PulseError("terminate must be contiguous int64")
        a = _lib.EvalArgs(body_pos=body_pos.data_ptr(), pos_env_stride=body_pos.stride(0), pos_body_stride=body_pos.stride(1),
                          body_pos_gt=body_pos_gt.data_ptr(), gt_env_stride=body_pos_gt.stride(0), gt_body_stride=body_pos_gt.stride(1),
                          terminate=terminate.data_ptr(), num_steps=self.num_steps.data_ptr(), num_envs=self.N, bound=self.bound,
                          max_steps_all=self.max_steps, ctrl=self.ctrl.data_ptr(), terminate_state=self.terminate_state.data_ptr(),
                          hist=self.hist.data_ptr(), sums=self.sums.data_ptr(), counts=self.counts.data_ptr(), mpjpe_out=self.mpjpe.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_eval_step(C.byref(a), _lib.current_stream(self.device)), "pulse_eval_step")

    def finished(self) -> bool:
        """Has the chunk ended (im_amp.py:275)?  Synchronises on a 4-byte read."""
        return bool(int(self.ctrl[1].item()))

    def read(self) -> Dict[str, np.ndarray]:
        return {"sums": self.sums.cpu().numpy(), "counts": self.counts.cpu().numpy(), "terminated": self.terminate_state.cpu().numpy().astype(bool),
                "steps": int(self.ctrl[0].item())}


def summarise(sums: np.ndarray, counts: np.ndarray, select: Optional[np.ndarray] = None) -> Dict[str, float]:
    """np.mean over the concatenated per-frame arrays of compute_metrics_lite = frame-weighted mean over the selected sequences, in mm."""
    if select is not None:
        sums, counts = sums[select], counts[select]
    out = {}
    for k, name in enumerate(METRIC_NAMES):
        c = counts[:, _COUNT_COL[k]].sum()
        out[name] = float(sums[:, k].sum() / c * 1000.0) if c > 0 else float("nan")
    return out


class EvalLoopB200:
    """`IMAmpAgent.eval` (im_amp.py:136-242) with the per-step bookkeeping on the device.

    Callbacks (the task / agent side, all device work, no return values needed):
        load_chunk(start_idx) -> (num_steps [N] ints, curr_ids [N] ints)   begin_seq_motion_samples / forward_motion_samples
                                                                           (humanoid_im.py:439-447): load clips start_idx.. in order
        reset_all()                                                         env_reset() of every env at motion time 0 (flags.test)
        step() -> (body_pos view, body_pos_gt, terminate_buf)               deterministic action + env step (+ reset of done envs)
    """

    def __init__(self, num_envs: int, num_unique: int, keys: Sequence[str], load_chunk: Callable, reset_all: Callable, step: Callable,
                 device="cuda:0", poll_every: int = 8, metrics=None):
        self.N, self.num_unique, self.keys = int(num_envs), int(num_unique), np.asarray(keys)
        self.load_chunk, self.reset_all, self.step_fn = load_chunk, reset_all, step
        # `metrics`: an object with the EvalMetricsB200 interface (begin_chunk / step / finished / read); the CPU suite injects a numpy
        # model of the device state machine to exercise this host loop without a GPU (tests/test_eval_host_cpu.py)
        self.metrics = metrics if metrics is not None else EvalMetricsB200(num_envs, device)
        self.poll_every = max(1, int(poll_every))

    def run(self) -> Dict:
        N, U = self.N, self.num_unique
        sums, counts, term = [], [], []
        start_idx, chunks, total_steps = 0, 0, 0
        while True:
            num_steps, curr_ids = self.load_chunk(start_idx)
            curr_ids = np.asarray(curr_ids)
            hit = np.flatnonzero(curr_ids == U - 1)
            bound = int(hit[0]) + 1 if hit.size > 0 else N                       # im_amp.py:254-256
            self.metrics.begin_chunk(num_steps, bound)
            self.reset_all()
            upper = int(np.max(num_steps)) + 2                                   # the stopping rule ends a chunk within max(num_steps) + 1 steps
            s = 0
            while s < upper:
                self.metrics.step(*self.step_fn())
                s += 1
                if s % self.poll_every == 0 and self.metrics.finished():
                    break
            r = self.metrics.read()
            total_steps += r["steps"]
            sums.append(r["sums"]); counts.append(r["counts"]); term.append(r["terminated"])
            chunks += 1
            if start_idx + N >= U:                                               # im_amp.py:295
                break
            start_idx += N                                                       # forward_motion_samples (humanoid_im.py:445-447)
        sums, counts, term = np.concatenate(sums)[:U], np.concatenate(counts)[:U], np.concatenate(term)[:U]
        success_rate = 1.0 - term.mean()                                         # :278
        all_print = summarise(sums, counts)
        succ_print = summarise(sums, counts, ~term) if (~term).any() else all_print   # :322-324
        info = {"eval_success_rate": float(success_rate), "eval_mpjpe_all": all_print["mpjpe_g"], "eval_mpjpe_succ": succ_print["mpjpe_g"],
                "accel_dist": succ_print["accel_dist"], "vel_dist": succ_print["vel_dist"], "mpjpel_all": all_print["mpjpe_l"],
                "mpjpel_succ": succ_print["mpjpe_l"], "mpjpe_pa": succ_print["mpjpe_pa"]}      # :333-342
        return {"eval_info": info, "failed_keys": self.keys[term], "success_keys": self.keys[~term], "terminated": term,
                "chunks": chunks, "steps": total_steps, "per_sequence": {"sums": sums, "counts": counts}}


def update_training_data(motion_dataset, failed_keys, auto_pmcp: bool = False, auto_pmcp_soft: bool = False) -> None:
    """IMAmpAgent.update_training_data (im_amp.py:126-132) on a MotionDatasetB200: hard / soft negative mining of the failed clips."""
    if auto_pmcp:
        motion_dataset.update_hard_sampling_weight(list(failed_keys))
    elif auto_pmcp_soft:
        motion_dataset.update_soft_sampling_weight(list(failed_keys))
