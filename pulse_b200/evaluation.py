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
load chunk), so it runs in front of Isaac Gym, of the stand-in task of the tests, or of a synthetic simulator.  `EvalStepsB200` is the
pass of a training driver (`PlayStepsB200`: HumanoidIm, `ImZStepsB200`: the VR task, `DistillStepsB200`: the PULSE student of
HumanoidImDistillGetup): its policy acts deterministically on the simulator tensors of the driver through the existing kernels,
chunk after chunk of a `MotionDatasetB200`, with `EvalLoopB200` as the chunk loop.  `eval_config` / `eval_settings` are the settings of the pass (im_amp.py:160-182) on a step configuration / on a live task.
"""
import contextlib
import dataclasses
import ctypes as C
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .rollout import GraphRunner

EVAL_TERMINATION_DISTANCE = 0.5                                                # im_amp.py:174 (UHC's termination distance)
ALL_BODIES = tuple(range(24))                  # `_eval_track_bodies_id` of the default `_eval_bodies`: every body (humanoid.py:388)
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
    or, in place of `step`,
        steps()                                                             the next `poll_every` evaluation steps, each ending with
                                                                            its `metrics.step` (device work only: a CUDA graph can hold it)
    """

    def __init__(self, num_envs: int, num_unique: int, keys: Sequence[str], load_chunk: Callable, reset_all: Callable,
                 step: Optional[Callable] = None, device="cuda:0", poll_every: int = 8, metrics=None, steps: Optional[Callable] = None):
        if (step is None) == (steps is None):
            raise _lib.PulseError("EvalLoopB200 takes one of step / steps")
        self.N, self.num_unique, self.keys = int(num_envs), int(num_unique), np.asarray(keys)
        self.load_chunk, self.reset_all, self.step_fn, self.steps_fn = load_chunk, reset_all, step, steps
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
            self.metrics.begin_chunk(num_steps, chunk_bound(curr_ids, U))
            self.reset_all()
            upper = int(np.max(num_steps)) + 2                                   # the stopping rule ends a chunk within max(num_steps) + 1 steps
            s = 0
            while s < upper:
                if self.steps_fn is not None:
                    self.steps_fn()                                              # steps past the end of the chunk are no-ops in the kernel
                    s += self.poll_every
                else:
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


def chunk_clip_ids(start_idx: int, num_envs: int, num_unique: int) -> np.ndarray:
    """The clips of the chunk that starts at `start_idx`, env by env: `torch.remainder(arange(N) + start_idx, U)` (motion_lib_base.py:208)."""
    return np.remainder(np.arange(int(num_envs)) + int(start_idx), int(num_unique))


def chunk_bound(curr_ids, num_unique: int) -> int:
    """Envs [0, bound) hold the chunk's distinct clips: up to and including the env of the last clip when the chunk wraps, else all
    (im_amp.py:254-256)."""
    curr_ids = np.asarray(curr_ids)
    hit = np.flatnonzero(curr_ids == int(num_unique) - 1)
    return int(hit[0]) + 1 if hit.size > 0 else int(curr_ids.shape[0])


def chunk_starts(num_envs: int, num_unique: int) -> List[int]:
    """`start_idx` of every chunk of a pass: 0 (begin_seq_motion_samples), then + N (forward_motion_samples, humanoid_im.py:439-447)
    until the chunk with start_idx + N >= U, the last one (im_amp.py:295)."""
    out = [0]
    while out[-1] + int(num_envs) < int(num_unique):
        out.append(out[-1] + int(num_envs))
    return out


def eval_config(cfg, strict_eval: bool = False, eval_body_ids: Sequence[int] = ALL_BODIES):
    """The `ImConfig` of an evaluation pass from the training one (im_amp.py:160-182): termination distance 0.5, the mean-distance reset
    criterion (`flags.im_eval and not strict_eval`), no cycle_motion, and the reset bodies swapped for `_eval_track_bodies_id` when there
    are more than 15 (full-body tracking; the three-point VR task keeps its own)."""
    reset_ids = tuple(int(j) for j in cfg.reset_body_ids)
    return dataclasses.replace(cfg, termination_distance=EVAL_TERMINATION_DISTANCE, use_mean_reset=not bool(strict_eval), cycle_motion=False,
                               reset_body_ids=tuple(int(j) for j in eval_body_ids) if len(reset_ids) > 15 else reset_ids)


@contextlib.contextmanager
def eval_settings(task, flags=None):
    """`IMAmpAgent.eval`'s settings on a live task for the duration of a pass (im_amp.py:160-182), put back afterwards (:220-233):
    `_termination_distances` 0.5, `cycle_motion` and `zero_out_far` off, the getup probabilities 0 (HumanoidImGetup), `_reset_bodies_id`
    -> `_eval_track_bodies_id` when there are more than 15, `flags.test` / `flags.im_eval` on (off afterwards, as the reference leaves
    them).  `flags`: the reference's flags object (`flags_compat.reference_flags()` when None); without one the task's `_pulse_im_eval`
    carries `im_eval` for `flags_compat.im_eval_mean_reset`."""
    from .flags_compat import reference_flags
    fl = flags if flags is not None else reference_flags()
    saved = dict(_termination_distances=task._termination_distances.clone(), cycle_motion=task.cycle_motion,
                 zero_out_far=getattr(task, "zero_out_far", False), _reset_bodies_id=task._reset_bodies_id,
                 _pulse_im_eval=getattr(task, "_pulse_im_eval", False))
    getup = "_recovery_episode_prob" in task.__dict__
    if getup:
        saved.update(_recovery_episode_prob=task._recovery_episode_prob, _fall_init_prob=task._fall_init_prob)
        task._recovery_episode_prob, task._fall_init_prob = 0, 0
    task._termination_distances[:] = EVAL_TERMINATION_DISTANCE
    task.cycle_motion, task.zero_out_far = False, False
    if fl is not None:
        fl.test, fl.im_eval = True, True
    task._pulse_im_eval = True
    if len(task._reset_bodies_id) > 15:
        task._reset_bodies_id = task._eval_track_bodies_id
    try:
        yield task
    finally:
        task._termination_distances[:] = saved.pop("_termination_distances")
        for k, v in saved.items():
            setattr(task, k, v)
        if fl is not None:
            fl.test, fl.im_eval = False, False


def update_training_data(motion_dataset, failed_keys, auto_pmcp: bool = False, auto_pmcp_soft: bool = False) -> None:
    """IMAmpAgent.update_training_data (im_amp.py:126-132) on a MotionDatasetB200: hard / soft negative mining of the failed clips."""
    if auto_pmcp:
        motion_dataset.update_hard_sampling_weight(list(failed_keys))
    elif auto_pmcp_soft:
        motion_dataset.update_soft_sampling_weight(list(failed_keys))


def driver_kind(driver) -> str:
    """The policy an `EvalStepsB200` pass runs for `driver`: "im" (PlayStepsB200, the actor's mean), "vr" (ImZStepsB200, the latent
    policy's mean through the frozen prior and decoder) or "distill" (DistillStepsB200, the VAE student at its posterior mean)."""
    from .distill import DistillStepsB200
    from .imz_rollout import ImZStepsB200
    from .rollout import PlayStepsB200
    if isinstance(driver, ImZStepsB200):
        return "vr"
    if isinstance(driver, PlayStepsB200):
        return "im"
    if isinstance(driver, DistillStepsB200):
        return "distill"
    raise _lib.PulseError(f"EvalStepsB200 evaluates PlayStepsB200 and ImZStepsB200 (the imitation and VR policies) and DistillStepsB200 "
                          f"(the distillation student), not {type(driver).__name__}")


class EvalStepsB200(GraphRunner):
    """One `IMAmpAgent.eval` pass (im_amp.py:136-242) of a training driver's policy over all `num_unique` clips of a `MotionDatasetB200`,
    on the driver's simulator tensors and step configuration: `PlayStepsB200` (HumanoidIm, im.yaml), `ImZStepsB200` (HumanoidImZ,
    pulse_z_vr.yaml) or `DistillStepsB200` (HumanoidImDistillGetup, env_im_vae.yaml + im_z_fit.yaml: the VAE student).  `EvalLoopB200`
    is the chunk loop; this class supplies its callbacks:
        load_chunk(start_idx)  `dataset.load_motions(N, random_sample=False, start_idx, eval_mode=True)`: clips (start_idx + e) % U, no
                               heading draw; a new MotionLibB200 and a new step compute over it with `eval_config`'s settings;
        reset_all()            every env at motion time 0 (`flags.test`): `pulse_reset_ref_state` with the start-time phase injected as 0,
                               then the observation of the reset envs;
        steps()                `poll_every` evaluation steps, each:
                                 1. the reset of the envs done at the previous step (again at motion time 0, im_amp.py:202);
                                 2. the deterministic action: HumanoidIm: the actor's mu on the normalised observation, `pulse_pd_targets`;
                                    VR task: z = prior_mu + mu (`pulse_latent_post` with zero noise), the frozen decoder, `pulse_pd_targets`;
                                    student: `eval_actor(use_mean=True)` -- z = vae_mu (amp_network_z_builder.py:94-95), the decoder --
                                    and `pulse_pd_targets`; the teacher is not run (humanoid_im_distill.py:152, flags.test);
                                 3. the `physics(t)` hook (it applies `pd_tar`);
                                 4. the fused step (`pulse_im_step` / `pulse_im_track_step`, STEP_ALL | STEP_ADVANCE) with the eval settings;
                                 5. `body_pos_gt` = MotionLibB200's query at progress * dt + start + offset after the step, the time the
                                    reward used (humanoid_im.py:667-671), and `pulse_eval_step` on the rigid-body view, `body_pos_gt`
                                    and `terminate_buf`.
    Launch structure: without hooks the `poll_every` steps are one CUDA graph and the host reads the 4-byte finished flag once per graph;
    with `physics` (or the `record(body_pos, body_pos_gt, terminate)` frame hook) every step is two graph segments, steps 1-2 and 4-5,
    around the hooks.  The graphs of a chunk are captured against that chunk's MotionLib (its handle is a launch argument), so every
    chunk captures its own.  `use_graphs=False` runs the same calls eagerly.
    Isolation: the pass keeps its own task-side state (progress, clip ids, start times, offsets, reset / terminate flags, observation,
    PD targets) and shares only the simulator tensors and the policy's evaluation workspaces with the driver.  No running statistic
    moves (the observation normaliser is read in evaluation mode; no value, AMP or optimiser state is touched) and the driver's graphs,
    buffers and MotionLib stay as they are.  Afterwards every env is reset into training through the driver's reset (im_amp.py:234)
    and the training observation is written to the driver's `obs_carry`.
    The student's pass needs no getup state of its own: at the pass's getup probabilities 0 (im_amp.py:167-172) every reset is a
    reference-state episode that zeroes the recovery counter, so the recovery masking never fires and the pass is the HumanoidIm
    pass; the driver's getup tensors (recovery counter, fall pool and its assignments) are not touched.  Its reset into training
    is the getup reset with the training probabilities, after the pass's last terminate flags are copied into the driver's
    `terminate_buf`: the recovery episodes fall on the envs the pass terminated."""

    def __init__(self, driver, physics: Optional[Callable[[int], None]] = None, poll_every: int = 8, use_graphs: bool = True,
                 strict_eval: bool = False, eval_body_ids: Sequence[int] = ALL_BODIES):
        self.kind = driver_kind(driver)
        self.vr = self.kind == "vr"
        self.driver, self.sim = driver, driver.sim
        self.policy = driver.vae if self.kind == "distill" else driver.policy
        self.dev, n = driver.dev, int(driver.n)
        self.n = n
        self.cfg = eval_config(driver.comp.cfg, strict_eval, eval_body_ids)
        self.physics, self.record = physics, None
        self.poll_every, self.use_graphs = max(1, int(poll_every)), bool(use_graphs)
        self.lib = _lib.load()
        dev = self.dev
        z = lambda *s, **k: torch.zeros(*s, device=dev, **k)
        # task-side state of the pass: `_sampled_motion_ids` is arange(num_envs) (humanoid_im.py:107), env e plays clip e of the chunk
        self.progress_buf, self.motion_ids = z(n, dtype=torch.int64), torch.arange(n, dtype=torch.int64, device=dev)
        self.motion_start_times, self.motion_start_offset, self.global_offset = z(n), z(n), z(n, 3)
        self.reset_buf, self.terminate_buf = z(n, dtype=torch.int64), z(n, dtype=torch.int64)
        self.phase = z(n)                                                       # flags.test: motion_times[:] = 0 (humanoid_im.py:976-977)
        self.obs, self.rew = z(n, driver.comp.obs_size), z(n)
        A = driver.pd[0].shape[0]
        self.pd_tar = z(n, A)
        if self.kind != "distill":                                               # the student's mu is a view of its decoder's workspace
            self.mus = z(n, self.policy.A)
        if self.vr:                                                              # pulse_latent_post's operands: zero noise, unused value
            E = self.policy.A
            self.eps, self.actions, self.neglogp = z(n, E), z(n, E), z(n)
            self.value, self.values = z(n, 1), z(n, 1)
        self.metrics = EvalMetricsB200(n, dev)
        self.comp = None
        self.body_pos_gt = None
        self._graphs, self._pool = {}, None

    # ------------------------------------------------------------------ the pieces of one step
    def _launch(self, name: str, *args) -> None:
        with torch.cuda.device(self.dev):
            _lib.check(getattr(self.lib, name)(*args, _lib.current_stream(self.dev)), name)

    def _state(self) -> dict:
        return dict(body_state=self.sim["body_state"], progress_buf=self.progress_buf, motion_ids=self.motion_ids,
                    motion_start_times=self.motion_start_times, motion_start_offset=self.motion_start_offset, global_offset=self.global_offset)

    def _reset(self) -> None:
        """env_reset(done_indices) at motion time 0 and the observation of the reset envs (Humanoid._reset_envs -> _compute_observations)."""
        s = self.sim
        self.comp.reset_envs(motion_ids=self.motion_ids, motion_start_times=self.motion_start_times, motion_start_offset=self.motion_start_offset,
                             global_offset=self.global_offset, progress_buf=self.progress_buf, root_states=s["root_states"], dof_pos=s["dof_pos"],
                             dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=self.reset_buf, terminate_buf=self.terminate_buf,
                             contact_forces=s.get("contact_forces"), actor_ids=s.get("actor_ids"), phase=self.phase, obs_buf=self.obs)

    def _act(self) -> None:
        """get_action(obs, is_determenistic=True) (im_amp.py:44-75) and the PD targets of pre_physics_step."""
        from .vae import pd_targets
        pol, d = self.policy, self.driver
        if self.kind == "distill":                                              # z = vae_mu (Z_MEAN), decoder; no teacher (flags.test)
            pd_targets(pol.eval_actor(self.obs, use_mean=True)["mus"], d.pd[0], d.pd[1], out=self.pd_tar, freeze=d.pd_freeze)
            return
        if not self.vr:
            pol.heads_into(self.obs, mus=self.mus, with_value=False)
            pd_targets(self.mus, d.pd[0], d.pd[1], out=self.pd_tar)
            return
        vae = d.vae
        prior_head, dec_in = vae.z_prior(self.obs)
        pol.heads_into(self.obs, mus=self.mus, with_value=False)
        a = _lib.LatentPostArgs(mu=self.mus.data_ptr(), ld_mu=self.mus.stride(0), logstd=pol.logstd.data_ptr(), eps=self.eps.data_ptr(),
                                ld_eps=self.eps.stride(0), latent=vae.E, actions=self.actions.data_ptr(), ld_actions=self.actions.stride(0),
                                neglogp=self.neglogp.data_ptr(), ld_neglogp=1, value=self.value.data_ptr(), ld_value=1,
                                values_out=self.values.data_ptr(), ld_values=1, prior_mu=prior_head.data_ptr(), ld_prior=prior_head.stride(0),
                                z_bf16=dec_in.data_ptr(), ld_z=dec_in.stride(0))
        self._launch("pulse_latent_post", C.byref(a), self.n)        # a_z = mu + exp(logstd) * 0 = mu; z = prior_mu + mu into the decoder operand
        pd_targets(vae.dec.forward(dec_in), d.pd[0], d.pd[1], out=self.pd_tar, freeze=d.pd_freeze)

    def _pre(self) -> None:
        self._reset()
        self._act()

    def _post(self) -> None:
        """post_physics_step with flags.im_eval (humanoid_im.py:662-673) and `_post_step_eval`'s device half (pulse_eval_step)."""
        s = self.sim
        self.comp.step(flags=_lib.STEP_ALL, advance=True, obs_buf=self.obs, rew_buf=self.rew, reset_buf=self.reset_buf,
                       terminate_buf=self.terminate_buf, dof_force=s.get("dof_force"), dof_vel=s["dof_vel"], **self._state())
        times = self.progress_buf * self.cfg.dt + self.motion_start_times + self.motion_start_offset
        self.body_pos_gt = self.comp.motion_lib.get_motion_state(self.motion_ids, times, offset=self.global_offset)["rg_pos"]
        self.metrics.step(s["body_state"][:, :, 0:3], self.body_pos_gt, self.terminate_buf)

    def _block(self) -> None:
        for _ in range(self.poll_every):
            self._pre()
            self._post()

    # ------------------------------------------------------------------ EvalLoopB200's callbacks
    def _load_chunk(self, start_idx: int):
        from .humanoid_im import HumanoidImCompute
        ds = self._dataset
        self._graphs, self._pool = {}, None                    # the previous chunk's graphs hold the previous MotionLib's handle
        self.comp = None
        lib = ds.load_motions(self.n, random_sample=False, start_idx=int(start_idx), eval_mode=True)
        self.comp = HumanoidImCompute(lib, self.cfg)
        self._t = 0
        return lib.get_motion_num_steps().cpu().numpy(), np.asarray(ds._curr_motion_ids)

    def _reset_all(self) -> None:
        self.reset_buf.fill_(1)
        self._reset()

    def _steps(self) -> None:
        if self.physics is None and self.record is None:
            self._run(("block",), self._block)
            self._t += self.poll_every
            return
        s = self.sim
        for _ in range(self.poll_every):
            self._run(("pre",), self._pre)
            if self.physics is not None:
                self.physics(self._t)
            self._run(("post",), self._post)
            if self.record is not None:
                self.record(s["body_state"][:, :24, 0:3], self.body_pos_gt, self.terminate_buf)
            self._t += 1

    def _reset_training(self) -> None:
        """`self.env_reset()` after the pass (im_amp.py:234): every env through the driver's own reset (training settings, its MotionLib,
        Philox start times keyed on a fresh offset), its observation into the driver's `obs_carry`."""
        d, s = self.driver, self.sim
        d.reset_buf.fill_(1)
        if self.vr:
            d._reset(0)
            if d.refresh is not None:
                d.refresh(0, d.reset_ws)
            ws = d.reset_ws
            d.comp.step(flags=_lib.STEP_OBS, obs_buf=d.obs_carry, env_ids=ws["env_list"], env_count=ws["count"], **d._state())
        elif self.kind == "distill":
            # the getup reset with the training probabilities: recovery episodes fall on the envs the pass's last step terminated
            # (`_reset_actors` reads `_terminate_buf`, humanoid_im_getup.py:135-162) and keep the state the pass left them in
            d.terminate_buf.copy_(self.terminate_buf)
            d._reset(0)
            if d.refresh is not None:
                d.refresh(0, d.reset_ws)
            ws = d.reset_ws
            d.comp.step(body_state=s["body_state"], progress_buf=s["progress_buf"], motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"],
                        motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"], obs_buf=d.obs_carry,
                        env_ids=ws["env_list"][:d.n], env_count=ws["count"], flags=_lib.STEP_OBS)
        else:
            d.comp.reset_envs(motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                              global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
                              dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=d.reset_buf, terminate_buf=d.terminate_buf,
                              cycle_counter=s.get("cycle_counter"), contact_forces=s.get("contact_forces"), amp_obs_buf=d.amp_init,
                              actor_ids=s.get("actor_ids"), seed=d.reset_seed, offset=0, offset_dev=d.policy.rng_offset, obs_buf=d.obs_carry,
                              amp_fresh=d.amp_fresh)
        self.policy.advance_rng(1)                             # the reset's draws above used block `rng_offset + 0`

    # ------------------------------------------------------------------ the pass
    def run(self, dataset, auto_pmcp: bool = False, auto_pmcp_soft: bool = False) -> Dict:
        """The pass over every clip of `dataset`, then the reset into training and, with `auto_pmcp` / `auto_pmcp_soft`,
        `update_training_data` (im_amp.py:126-132, :236).  Returns EvalLoopB200.run's result (`eval_info` with the reference's eight keys,
        `failed_keys`, `success_keys`, `terminated`, `chunks`, `steps`, `per_sequence`) plus `termination_history`, the dataset's
        PMCP failure counts after the update."""
        self._dataset = dataset
        loop = EvalLoopB200(self.n, dataset._num_unique_motions, dataset._motion_data_keys, load_chunk=self._load_chunk,
                            reset_all=self._reset_all, steps=self._steps, device=self.dev, poll_every=self.poll_every, metrics=self.metrics)
        try:
            out = loop.run()
        finally:
            self._dataset, self.comp = None, None
            self._graphs, self._pool = {}, None
        self._reset_training()
        update_training_data(dataset, out["failed_keys"], auto_pmcp, auto_pmcp_soft)
        out["termination_history"] = dataset._termination_history.clone()
        return out
