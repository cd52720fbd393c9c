"""HumanoidIm per-step compute on the GPU: host-side mirror of the reference task's
`_compute_reward` / `_compute_reset` / `_compute_observations` / `_compute_amp_observations`
(phc/env/tasks/humanoid_im.py, humanoid.py, humanoid_amp.py), backed by the fused CUDA kernels.

Two layers:
  * `HumanoidImCompute` -- explicit-tensor API (what bench.py, the tests and the mixin call);
  * `HumanoidImB200Mixin` -- drop-in overrides with the reference's method names, to be mixed in
    front of `phc.env.tasks.humanoid_im.HumanoidIm` (see INTEGRATION.md); Isaac Gym keeps doing the
    physics and owns the state tensors, which are read in place through their strides;
  * `HumanoidImGetupB200Mixin` -- the same for `HumanoidImGetup`, whose getup reset it serves too.

Everything runs on torch's current CUDA stream; no host synchronisation is added (the reference's
MotionLib-cache compare, humanoid_im.py:952-953, costs one D2H sync per call and is gone).
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .motion_lib import MotionLibB200

NUM_BODIES, NUM_DOF = 24, 69
SELF_OBS, TASK_OBS, AMP_OBS = 358, 576, 196
IM_OBS = SELF_OBS + TASK_OBS
DEFAULT_RESET_BODIES = tuple(j for j in range(24) if j not in (3, 4, 7, 8))  # env_im.yaml:38
# dt = control_freq_inv * sim dt, with sim dt a C float inside Isaac Gym: 2 * fp32(1/60)
STEP_DT = float(torch.tensor(1.0 / 60.0, dtype=torch.float32) * 2)


@dataclass
class ImConfig:
    """The subset of cfg['env'] the step path reads (humanoid_im.py:36-110, humanoid.py:254-349)."""
    dt: float = STEP_DT
    reward_specs: Dict[str, float] = field(default_factory=lambda: {
        "k_pos": 100.0, "k_rot": 10.0, "k_vel": 0.1, "k_ang_vel": 0.1, "w_pos": 0.5, "w_rot": 0.3, "w_vel": 0.1, "w_ang_vel": 0.1})
    power_reward: bool = True
    power_coefficient: float = 0.0005
    reset_body_ids: Sequence[int] = DEFAULT_RESET_BODIES
    termination_distance: float = 0.25
    enable_early_termination: bool = True
    cycle_motion: bool = False
    max_episode_length: int = 300
    use_mean_reset: bool = False     # flags.im_eval and not strict_eval
    num_amp_obs_steps: int = 10
    track_body_ids: Optional[Sequence[int]] = None   # _track_bodies_id: None = all 24 bodies, the 934-float row
    obs_version: int = 6             # obs_v of the tracked row: 6 or 7 (humanoid_im.py:1328-1413)


TRACK_BLOCKS = {6: ((0, 3), (72, 6), (216, 3), (288, 3), (360, 3), (432, 6)), 7: ((0, 3), (216, 3), (360, 3))}   # (offset, width) in v6


def track_columns(version: int, track_ids: Sequence[int]) -> torch.Tensor:
    """Column of the full-body v6 task block (576 floats) behind each column of the tracked task block: v6 and v7 of a body subset are
    column selections of the full v6 pieces, block-major over the bodies in `track_ids` order."""
    if int(version) not in TRACK_BLOCKS:
        raise _lib.PulseError(f"tracked observation version {version}: have 6 and 7")
    return torch.tensor([off + w * int(j) + c for off, w in TRACK_BLOCKS[int(version)] for j in track_ids for c in range(w)], dtype=torch.int64)


def _strided(t: torch.Tensor, inner: int):
    """(data_ptr, env stride in floats) of a [N, inner...] float32 view whose rows are contiguous runs."""
    if t.dtype != torch.float32:
        raise _lib.PulseError(f"expected float32 state tensor, got {t.dtype}")
    return t.data_ptr(), t.stride(0)


class HumanoidImCompute:
    def __init__(self, motion_lib: MotionLibB200, cfg: Optional[ImConfig] = None):
        if getattr(motion_lib, "smplx", False):
            raise _lib.PulseError("HumanoidImCompute serves the 24-body SMPL humanoid; the MotionLib holds 52-body SMPL-X tables")
        self.lib = _lib.load()
        self.motion_lib = motion_lib
        self.cfg = cfg or ImConfig()
        self.device = motion_lib._device
        self.termination_distances = torch.full((NUM_BODIES,), float(self.cfg.termination_distance), device=self.device)
        self.reset_body_mask = 0
        for j in self.cfg.reset_body_ids:
            self.reset_body_mask |= 1 << int(j)
        self.track = None
        ids = self.cfg.track_body_ids
        if ids is not None:
            ids = [int(j) for j in ids]
            if not ids or len(set(ids)) != len(ids) or not all(0 <= j < NUM_BODIES for j in ids):
                raise _lib.PulseError(f"track_body_ids must be distinct body ids in [0, {NUM_BODIES}), got {ids}")
            if int(self.cfg.obs_version) not in TRACK_BLOCKS:
                raise _lib.PulseError(f"tracked observation version {self.cfg.obs_version}: have 6 and 7")
            self.track = _lib.ImTrack(num_track=len(ids), version=int(self.cfg.obs_version))
            for j in range(NUM_BODIES):
                self.track.rank[j] = ids.index(j) if j in ids else -1

    @classmethod
    def from_task(cls, task, **cfg) -> "HumanoidImCompute":
        """The compute of a live HumanoidIm task: its MotionLib (packed once), step dt, reward, reset and AMP settings and termination
        distances; `cfg` sets further ImConfig fields (the tracked observation)."""
        ml = task._motion_lib
        motion_lib = ml if isinstance(ml, MotionLibB200) else MotionLibB200.from_reference(ml, device=task.device)
        c = ImConfig(
            dt=float(torch.tensor(task.dt, dtype=torch.float32)), reward_specs={k: float(v) for k, v in task.reward_specs.items()},
            power_reward=bool(task.power_reward), power_coefficient=float(task.power_coefficient),
            reset_body_ids=tuple(int(i) for i in task._reset_bodies_id.tolist()),
            enable_early_termination=bool(task._enable_early_termination), cycle_motion=bool(task.cycle_motion),
            max_episode_length=int(task.max_episode_length), num_amp_obs_steps=int(getattr(task, "_num_amp_obs_steps", 10)), **cfg)
        comp = cls(motion_lib, c)
        comp.termination_distances = task._termination_distances.reshape(-1)[:NUM_BODIES].to(task.device, torch.float32).contiguous()
        return comp

    @property
    def obs_size(self) -> int:
        """Floats of the observation row `step` writes: 934, or 358 + 24 K (v6) / 358 + 9 K (v7) for K tracked bodies."""
        if self.track is None:
            return IM_OBS
        return SELF_OBS + sum(w for _, w in TRACK_BLOCKS[self.track.version]) * self.track.num_track

    # ------------------------------------------------------------------------------------------
    def step(self, *, body_state: torch.Tensor, progress_buf: torch.Tensor, motion_ids: torch.Tensor,
             motion_start_times: torch.Tensor, motion_start_offset: torch.Tensor, global_offset: torch.Tensor,
             dof_vel: Optional[torch.Tensor] = None, dof_force: Optional[torch.Tensor] = None,
             cycle_counter: Optional[torch.Tensor] = None, obs_buf: Optional[torch.Tensor] = None,
             self_obs_buf: Optional[torch.Tensor] = None, rew_buf: Optional[torch.Tensor] = None,
             reward_raw: Optional[torch.Tensor] = None, reset_buf: Optional[torch.Tensor] = None,
             terminate_buf: Optional[torch.Tensor] = None, pass_time: Optional[torch.Tensor] = None,
             ref_body_pos=None, ref_body_vel=None, ref_body_rot=None, ref_dof_pos=None,
             env_ids: Optional[torch.Tensor] = None, flags: int = _lib.STEP_ALL, num_envs: Optional[int] = None,
             env_count: Optional[torch.Tensor] = None, recovery_counter: Optional[torch.Tensor] = None,
             fdones_out: Optional[torch.Tensor] = None, advance: bool = False) -> None:
        """One fused launch.  `body_state` is the [N, bodies_per_env, 13] rigid-body-state view (or its
        [:, :24] slice); `dof_vel` may be the strided Isaac Gym view dof_state[..., 1].  With `track_body_ids` configured the
        observation row is the tracked one (`obs_size` floats, `pulse_im_track_step`); reward and reset stay full-body."""
        c = self.cfg
        a = _lib.ImStepArgs()
        if body_state.dim() != 3 or body_state.shape[-1] != 13 or body_state.stride(-1) != 1 or body_state.stride(1) != 13:
            raise _lib.PulseError(f"body_state must be a [N,B,13] view with row stride 13, got {tuple(body_state.shape)} / {body_state.stride()}")
        a.body_state, a.body_env_stride = _strided(body_state, 13)
        n_total = body_state.shape[0]
        use_power = c.power_reward and (flags & _lib.STEP_REWARD) and dof_force is not None
        if use_power:
            if dof_vel is None:
                raise _lib.PulseError("power reward needs dof_vel")
            a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_vel.data_ptr(), dof_vel.stride(0), dof_vel.stride(1)
            a.dof_force, a.dof_force_stride = dof_force.data_ptr(), dof_force.stride(0)
            if dof_force.stride(1) != 1:
                raise _lib.PulseError("dof_force rows must be contiguous")
        for name, t, dt_ in (("progress_buf", progress_buf, torch.int64), ("motion_ids", motion_ids, torch.int64),
                             ("motion_start_times", motion_start_times, torch.float32),
                             ("motion_start_offset", motion_start_offset, torch.float32), ("global_offset", global_offset, torch.float32)):
            if t.dtype != dt_ or not t.is_contiguous() or t.shape[0] != n_total:
                raise _lib.PulseError(f"{name}: expected contiguous {dt_} with {n_total} rows, got {t.dtype} {tuple(t.shape)}")
            setattr(a, name, t.data_ptr())
        if cycle_counter is not None:
            if cycle_counter.dtype != torch.int32:
                raise _lib.PulseError("cycle_counter must be int32 (humanoid_im.py:71)")
            a.cycle_counter = cycle_counter.data_ptr()
        a.termination_distances = self.termination_distances.data_ptr()
        a.reset_body_mask = self.reset_body_mask
        a.flags = flags
        a.dt = c.dt
        for k, v in c.reward_specs.items():
            setattr(a, k, float(v))
        a.power_coefficient = c.power_coefficient
        a.cycle_motion = int(c.cycle_motion)
        a.max_episode_length = int(c.max_episode_length)
        a.enable_early_termination = int(c.enable_early_termination)
        a.use_mean_reset = int(c.use_mean_reset)
        if flags & _lib.STEP_OBS:
            if obs_buf is None or obs_buf.dtype != torch.float32 or obs_buf.stride(-1) != 1 or obs_buf.shape[-1] < self.obs_size:
                raise _lib.PulseError(f"obs_buf must be float32 [N, >={self.obs_size}] with contiguous rows")
            a.obs_buf, a.obs_stride = obs_buf.data_ptr(), obs_buf.stride(0)
            if self_obs_buf is not None:
                a.self_obs_buf = self_obs_buf.data_ptr()
            for name, t in (("ref_body_pos", ref_body_pos), ("ref_body_vel", ref_body_vel), ("ref_body_rot", ref_body_rot),
                            ("ref_dof_pos", ref_dof_pos)):
                if t is not None:
                    if not t.is_contiguous():
                        raise _lib.PulseError(f"{name} must be contiguous")
                    setattr(a, name, t.data_ptr())
        if flags & _lib.STEP_REWARD:
            a.rew_buf = rew_buf.data_ptr()
            if reward_raw is not None:
                a.reward_raw, a.raw_stride = reward_raw.data_ptr(), reward_raw.stride(0)
        if flags & _lib.STEP_RESET:
            if reset_buf.dtype != torch.int64 or terminate_buf.dtype != torch.int64:
                raise _lib.PulseError("reset_buf / terminate_buf must be int64 (base_task.py:99-105)")
            a.reset_buf, a.terminate_buf = reset_buf.data_ptr(), terminate_buf.data_ptr()
        if pass_time is not None:
            a.pass_time = pass_time.data_ptr()
        n = n_total if num_envs is None else num_envs
        if env_ids is not None:
            if env_ids.dtype != torch.int64 or not env_ids.is_contiguous():
                raise _lib.PulseError("env_ids must be contiguous int64")
            a.env_ids = env_ids.data_ptr()
            n = int(env_ids.shape[0])
            if env_count is not None:                 # device-side list length (reset path): never read on the host
                if env_count.dtype != torch.int32 or env_count.numel() < 1:
                    raise _lib.PulseError("env_count must be an int32 device scalar")
                a.env_count = env_count.data_ptr()
        if recovery_counter is not None:              # HumanoidImGetup (humanoid_im_getup.py:203-210)
            if recovery_counter.dtype != torch.int32 or not recovery_counter.is_contiguous():
                raise _lib.PulseError("recovery_counter must be contiguous int32")
            a.recovery_counter, a.progress_rw = recovery_counter.data_ptr(), progress_buf.data_ptr()
        if fdones_out is not None:
            if fdones_out.dtype != torch.float32 or not fdones_out.is_contiguous():
                raise _lib.PulseError("fdones_out must be contiguous float32 [N]")
            a.fdones_out = fdones_out.data_ptr()
        if advance:                                   # `self.progress_buf += 1` (humanoid.py:1317) inside the launch
            a.flags = flags | _lib.STEP_ADVANCE
            a.progress_rw = progress_buf.data_ptr()
        with torch.cuda.device(self.device):
            if self.track is None:
                _lib.check(self.lib.pulse_im_step(self.motion_lib.handle, C.byref(a), n, _lib.current_stream(self.device)), "pulse_im_step")
            else:
                _lib.check(self.lib.pulse_im_track_step(self.motion_lib.handle, C.byref(a), C.byref(self.track), n, _lib.current_stream(self.device)),
                           "pulse_im_track_step")

    # ------------------------------------------------------------------------------------------
    def amp_obs(self, *, body_state: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, amp_obs_buf: torch.Tensor,
                shift_history: bool = True) -> None:
        """humanoid_amp.py:622-630 + :632-667 in one launch; amp_obs_buf [N, steps, 196] updated in place."""
        a = _lib.AmpObsArgs()
        a.body_state, a.body_env_stride = _strided(body_state, 13)
        if dof_pos.stride() != dof_vel.stride():
            raise _lib.PulseError("dof_pos and dof_vel must share strides (views of one dof-state tensor)")
        a.dof_pos, a.dof_vel = dof_pos.data_ptr(), dof_vel.data_ptr()
        a.dof_env_stride, a.dof_elem_stride = dof_pos.stride(0), dof_pos.stride(1)
        if not amp_obs_buf.is_contiguous() or amp_obs_buf.shape[-1] != AMP_OBS:
            raise _lib.PulseError("amp_obs_buf must be contiguous [N, steps, 196]")
        a.amp_obs_buf = amp_obs_buf.data_ptr()
        a.num_steps = int(amp_obs_buf.shape[1])
        a.shift_history = int(shift_history)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_amp_obs(C.byref(a), int(body_state.shape[0]), _lib.current_stream(self.device)), "pulse_amp_obs")


    def amp_obs_row(self, *, body_state: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, prev: torch.Tensor, out: torch.Tensor,
                    fresh: Optional[torch.Tensor] = None, fresh_rows: Optional[torch.Tensor] = None) -> None:
        """This step's AMP observation row of every env, [current 196 | the previous row's first (steps-1)*196 floats], written straight
        into its experience slice `out` [N, steps*196] (any row stride) from the previous step's slice `prev` -- `_update_hist_amp_obs`
        + `_compute_amp_observations` + the experience-buffer copy (humanoid_amp.py:622-667, amp_agent.py:385) without moving the
        history twice.  Envs flagged in `fresh` (set by `reset_envs`) take their history from `fresh_rows` [N, steps, 196]."""
        a = _lib.AmpRowArgs()
        a.body_state, a.body_env_stride = _strided(body_state, 13)
        if dof_pos.stride() != dof_vel.stride():
            raise _lib.PulseError("dof_pos and dof_vel must share strides (views of one dof-state tensor)")
        a.dof_pos, a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_pos.data_ptr(), dof_vel.data_ptr(), dof_pos.stride(0), dof_pos.stride(1)
        steps = out.shape[-1] // AMP_OBS
        if out.shape[-1] != steps * AMP_OBS or prev.shape != out.shape or out.stride(-1) != 1 or prev.stride(-1) != 1:
            raise _lib.PulseError("prev / out must be [N, steps*196] views with contiguous rows")
        a.prev, a.ld_prev, a.out, a.ld_out, a.num_steps = prev.data_ptr(), prev.stride(0), out.data_ptr(), out.stride(0), steps
        if fresh is not None:
            if fresh.dtype != torch.int32 or fresh_rows is None or not fresh_rows.is_contiguous():
                raise _lib.PulseError("fresh must be int32 [N] and come with contiguous fresh_rows [N, steps, 196]")
            a.fresh, a.fresh_rows = fresh.data_ptr(), fresh_rows.data_ptr()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_amp_obs_row(C.byref(a), int(body_state.shape[0]), _lib.current_stream(self.device)), "pulse_amp_obs_row")

    # ------------------------------------------------------------------------------------------
    def build_amp_obs_demo(self, motion_ids: torch.Tensor, motion_times0: torch.Tensor, num_steps: Optional[int] = None,
                           first_step: int = 0) -> torch.Tensor:
        """HumanoidAMP.build_amp_obs_demo (humanoid_amp.py:253-284): AMP observations of the reference motion at
        t0 - k*dt, k = 0..steps-1, one MotionLib query (no offset) + one AMP-obs launch.  Returns [n, steps*196]."""
        steps = int(num_steps or self.cfg.num_amp_obs_steps)
        n = int(motion_ids.shape[0])
        dev = self.device
        ids = motion_ids.to(dev).unsqueeze(-1).repeat(1, steps).reshape(-1)
        k = torch.arange(0, steps, device=dev)
        if first_step:   # _init_amp_obs_ref (humanoid_amp.py:540-541): -dt * (arange + 1)
            k = k + first_step
        times = (motion_times0.to(dev).unsqueeze(-1) + (-self.cfg.dt) * k).reshape(-1)
        ms = self.motion_lib.get_motion_state(ids, times)
        body = torch.cat([ms["rg_pos"], ms["rb_rot"], ms["body_vel"], ms["body_ang_vel"]], dim=-1).contiguous()   # [n*steps, 24, 13]
        out = torch.empty(n * steps, 1, AMP_OBS, device=dev)
        self.amp_obs(body_state=body, dof_pos=ms["dof_pos"], dof_vel=ms["dof_vel"], amp_obs_buf=out, shift_history=False)
        return out.view(n, steps * AMP_OBS)

    def _reset_args(self, ws, *, motion_ids, motion_start_times, motion_start_offset, global_offset, progress_buf, root_states, dof_pos,
                    dof_vel, rigid_body_state, reset_buf, env_ids, terminate_buf, cycle_counter, contact_forces, amp_obs_buf, actor_ids,
                    phase, seed, offset, amp_fresh, offset_dev) -> "_lib.ResetArgs":
        """Checks the reset set, the views and their strides, and fills pulse_reset_args_t (outputs: ws env_list / actor_list / count)."""
        N = int(progress_buf.shape[0])
        if (reset_buf is None) == (env_ids is None):
            raise _lib.PulseError("reset_envs takes either the reset_buf mask or an explicit env_ids list")
        if rigid_body_state.dim() != 3 or rigid_body_state.shape[-1] != 13 or rigid_body_state.stride(1) != 13 or rigid_body_state.stride(2) != 1:
            raise _lib.PulseError("rigid_body_state must be a [N,B,13] view with row stride 13")
        if dof_pos.stride() != dof_vel.stride():
            raise _lib.PulseError("dof_pos and dof_vel must share strides (views of one dof-state tensor)")
        a = _lib.ResetArgs()
        if reset_buf is not None:
            if reset_buf.dtype != torch.int64:
                raise _lib.PulseError("reset_buf must be int64")
            a.reset_buf = reset_buf.data_ptr()
        else:
            if env_ids.dtype != torch.int64 or not env_ids.is_contiguous():
                raise _lib.PulseError("env_ids must be contiguous int64")
            a.env_ids_in, a.num_ids = env_ids.data_ptr(), int(env_ids.shape[0])
        if phase is not None:
            if phase.dtype != torch.float32 or phase.shape[0] != N:
                raise _lib.PulseError("phase must be float32 [N] (one uniform draw per env)")
            a.phase = phase.data_ptr()
        a.seed, a.offset = int(seed) & (2 ** 64 - 1), int(offset) & (2 ** 64 - 1)
        for name, t, dt_ in (("motion_ids", motion_ids, torch.int64), ("motion_start_times", motion_start_times, torch.float32),
                             ("motion_start_offset", motion_start_offset, torch.float32), ("global_offset", global_offset, torch.float32),
                             ("progress_buf", progress_buf, torch.int64)):
            if t.dtype != dt_ or not t.is_contiguous() or t.shape[0] != N:
                raise _lib.PulseError(f"{name}: expected contiguous {dt_} with {N} rows")
            setattr(a, name, t.data_ptr())
        if cycle_counter is not None:
            a.cycle_counter = cycle_counter.data_ptr()
        if terminate_buf is not None:
            a.terminate_buf = terminate_buf.data_ptr()
        a.root_states, a.root_env_stride = root_states.data_ptr(), root_states.stride(0)
        a.dof_pos, a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_pos.data_ptr(), dof_vel.data_ptr(), dof_pos.stride(0), dof_pos.stride(1)
        a.rigid_body_state, a.body_env_stride = rigid_body_state.data_ptr(), rigid_body_state.stride(0)
        if contact_forces is not None:
            a.contact_forces, a.contact_env_stride, a.contact_bodies = contact_forces.data_ptr(), contact_forces.stride(0), int(contact_forces.shape[1])
        if amp_obs_buf is not None:
            if not amp_obs_buf.is_contiguous() or amp_obs_buf.shape[-1] != AMP_OBS:
                raise _lib.PulseError("amp_obs_buf must be contiguous [N, steps, 196]")
            a.amp_obs_buf, a.num_amp_steps = amp_obs_buf.data_ptr(), int(amp_obs_buf.shape[1])
        a.dt = self.cfg.dt
        if actor_ids is not None:
            if actor_ids.dtype != torch.int32:
                raise _lib.PulseError("actor_ids must be int32 (humanoid.py:590)")
            a.actor_ids = actor_ids.data_ptr()
        a.env_list, a.actor_list, a.count = ws["env_list"].data_ptr(), ws["actor_list"].data_ptr(), ws["count"].data_ptr()
        if amp_fresh is not None:
            if amp_fresh.dtype != torch.int32 or amp_fresh.shape[0] != N:
                raise _lib.PulseError("amp_fresh must be int32 [N]")
            a.amp_fresh = amp_fresh.data_ptr()
        if offset_dev is not None:                    # int64 / uint64 device counter added to `offset`
            a.offset_dev = offset_dev.data_ptr()
        return a

    def reset_envs(self, *, motion_ids: torch.Tensor, motion_start_times: torch.Tensor, motion_start_offset: torch.Tensor,
                   global_offset: torch.Tensor, progress_buf: torch.Tensor, root_states: torch.Tensor, dof_pos: torch.Tensor,
                   dof_vel: torch.Tensor, rigid_body_state: torch.Tensor, reset_buf: Optional[torch.Tensor] = None,
                   env_ids: Optional[torch.Tensor] = None, terminate_buf: Optional[torch.Tensor] = None,
                   cycle_counter: Optional[torch.Tensor] = None, contact_forces: Optional[torch.Tensor] = None,
                   amp_obs_buf: Optional[torch.Tensor] = None, actor_ids: Optional[torch.Tensor] = None,
                   phase: Optional[torch.Tensor] = None, seed: int = 0, offset: int = 0, obs_buf: Optional[torch.Tensor] = None,
                   self_obs_buf: Optional[torch.Tensor] = None, amp_fresh: Optional[torch.Tensor] = None,
                   offset_dev: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """The per-step env reset of the rollout loop (`self.obs = self.env_reset(done_indices)`, amp_agent.py:352 ->
        Humanoid.reset -> _reset_envs, humanoid.py:526-587, humanoid_amp.py:347-356, :468-488, :519-597, humanoid_im.py:921-989)
        WITHOUT a host round trip: `pulse_reset_ref_state` (device-side compaction of `reset_buf` -- or the explicit `env_ids` --
        start-time draw, MotionLib query, scatter into the simulator's root / dof / rigid-body views, counters cleared, AMP
        history back-filled) followed by the fused step kernel in observation mode on the compacted list.
        `phase`: per-ENV uniform draws (tests); None -> Philox4x32-10(seed, env, offset) inside the kernel.
        Returns {'env_list', 'actor_list', 'count'}: device tensors for gym.set_*_tensor_indexed (count stays on the device)."""
        N = int(progress_buf.shape[0])
        dev = self.device
        ws = getattr(self, "_reset_ws", None)
        if ws is None or ws["env_list"].shape[0] < N:
            ws = {"env_list": torch.zeros(N, dtype=torch.int64, device=dev), "actor_list": torch.zeros(N, dtype=torch.int32, device=dev),
                  "count": torch.zeros(1, dtype=torch.int32, device=dev)}
            self._reset_ws = ws
        a = self._reset_args(ws, motion_ids=motion_ids, motion_start_times=motion_start_times, motion_start_offset=motion_start_offset,
                             global_offset=global_offset, progress_buf=progress_buf, root_states=root_states, dof_pos=dof_pos,
                             dof_vel=dof_vel, rigid_body_state=rigid_body_state, reset_buf=reset_buf, env_ids=env_ids,
                             terminate_buf=terminate_buf, cycle_counter=cycle_counter, contact_forces=contact_forces,
                             amp_obs_buf=amp_obs_buf, actor_ids=actor_ids, phase=phase, seed=seed, offset=offset, amp_fresh=amp_fresh,
                             offset_dev=offset_dev)
        with torch.cuda.device(dev):
            _lib.check(self.lib.pulse_reset_ref_state(self.motion_lib.handle, C.byref(a), N, _lib.current_stream(dev)), "pulse_reset_ref_state")
        if obs_buf is not None:   # _compute_observations(env_ids) on the compacted list; its length stays on the device
            n_list = N if env_ids is None else int(env_ids.shape[0])
            self.step(body_state=rigid_body_state, progress_buf=progress_buf, motion_ids=motion_ids, motion_start_times=motion_start_times,
                      motion_start_offset=motion_start_offset, global_offset=global_offset, obs_buf=obs_buf, self_obs_buf=self_obs_buf,
                      env_ids=ws["env_list"][:n_list], env_count=ws["count"], flags=_lib.STEP_OBS)
        return ws

    def reset_getup(self, *, motion_ids: torch.Tensor, motion_start_times: torch.Tensor, motion_start_offset: torch.Tensor,
                    global_offset: torch.Tensor, progress_buf: torch.Tensor, root_states: torch.Tensor, dof_pos: torch.Tensor,
                    dof_vel: torch.Tensor, rigid_body_state: torch.Tensor, terminate_buf: torch.Tensor, recovery_counter: torch.Tensor,
                    available_fall_states: torch.Tensor, fall_id_assignments: torch.Tensor, fall_root_states: torch.Tensor,
                    fall_dof_pos: torch.Tensor, fall_dof_vel: torch.Tensor, recovery_prob: float, fall_prob: float, recovery_steps: int,
                    reset_buf: Optional[torch.Tensor] = None, env_ids: Optional[torch.Tensor] = None,
                    cycle_counter: Optional[torch.Tensor] = None, contact_forces: Optional[torch.Tensor] = None,
                    amp_obs_buf: Optional[torch.Tensor] = None, actor_ids: Optional[torch.Tensor] = None,
                    phase: Optional[torch.Tensor] = None, recovery_u: Optional[torch.Tensor] = None, fall_u: Optional[torch.Tensor] = None,
                    fall_keys: Optional[torch.Tensor] = None, seed: int = 0, offset: int = 0, amp_fresh: Optional[torch.Tensor] = None,
                    offset_dev: Optional[torch.Tensor] = None, check: bool = False) -> Dict[str, torch.Tensor]:
        """HumanoidImGetup's reset (`_reset_actors`, humanoid_im_getup.py:135-182, + `_reset_env_tensors`) for the envs of `reset_buf`
        or `env_ids`, in one `pulse_reset_getup` call and without a host round trip: recovery episodes (counter set, state kept), fall
        episodes (distinct free states of the fall pool copied in), reference-state episodes (exactly `reset_envs`'s device work).
        The getup tensors are the task's own, updated in place: `recovery_counter` (int32), `available_fall_states` /
        `fall_id_assignments` (int64; every assignment must index the pool), `fall_root_states` [P, 13], `fall_dof_pos` /
        `fall_dof_vel` [P, 69].
        Draws: `phase` / `recovery_u` / `fall_u` per ENV and `fall_keys` per fall state (uniforms, tests and the mixin inject them),
        or None -> Philox4x32-10(seed, index, offset [+ *offset_dev]) inside the kernels.
        The simulator refresh, the observation of the reset envs and `getup_amp_init` follow.  Returns device tensors: the union
        'env_list' / 'actor_list' / 'count' (as `reset_envs`), 'ref_list' / 'fall_list' / 'recovery_list' with 'class_counts' [3],
        'env_class' [N] (GETUP_REF / _FALL / _RECOVERY for the reset envs) and 'error', the number of fall envs that found no free
        state since the workspace was made (they take a reference-state episode; the reference asserts instead).  `check=True` reads
        that word -- one host synchronisation -- and raises PulseError when it is non-zero."""
        N = int(progress_buf.shape[0])
        P = int(fall_root_states.shape[0])
        dev = self.device
        ws = getattr(self, "_getup_ws", None)
        if ws is None or ws["env_list"].shape[0] != N or ws["fall_key_scratch"].shape[0] != P:
            i64 = lambda: torch.zeros(N, dtype=torch.int64, device=dev)
            ws = {"env_list": i64(), "actor_list": torch.zeros(N, dtype=torch.int32, device=dev), "count": torch.zeros(1, dtype=torch.int32, device=dev),
                  "ref_list": i64(), "fall_list": i64(), "recovery_list": i64(), "class_counts": torch.zeros(3, dtype=torch.int32, device=dev),
                  "env_class": torch.zeros(N, dtype=torch.uint8, device=dev), "error": torch.zeros(1, dtype=torch.int32, device=dev),
                  "fall_pick": i64(), "fall_key_scratch": torch.zeros(P, dtype=torch.int64, device=dev)}
            self._getup_ws = ws
        if terminate_buf is None:
            raise _lib.PulseError("reset_getup needs terminate_buf (it selects the recovery envs)")
        g = _lib.GetupResetArgs()
        g.base = self._reset_args(ws, motion_ids=motion_ids, motion_start_times=motion_start_times, motion_start_offset=motion_start_offset,
                                  global_offset=global_offset, progress_buf=progress_buf, root_states=root_states, dof_pos=dof_pos,
                                  dof_vel=dof_vel, rigid_body_state=rigid_body_state, reset_buf=reset_buf, env_ids=env_ids,
                                  terminate_buf=terminate_buf, cycle_counter=cycle_counter, contact_forces=contact_forces,
                                  amp_obs_buf=amp_obs_buf, actor_ids=actor_ids, phase=phase, seed=seed, offset=offset, amp_fresh=amp_fresh,
                                  offset_dev=offset_dev)
        if env_ids is not None and env_ids.numel() == 0:   # an empty tensor may have no storage: any device address serves num_ids = 0
            g.base.env_ids_in = ws["env_list"].data_ptr()
        for name, t, n in (("recovery_u", recovery_u, N), ("fall_u", fall_u, N), ("fall_keys", fall_keys, P)):
            if t is not None:
                if t.dtype != torch.float32 or not t.is_contiguous() or t.shape[0] != n:
                    raise _lib.PulseError(f"{name} must be contiguous float32 [{n}]")
                setattr(g, name, t.data_ptr())
        for name, t, dt_, n in (("recovery_counter", recovery_counter, torch.int32, N), ("available_fall_states", available_fall_states, torch.int64, P),
                                ("fall_id_assignments", fall_id_assignments, torch.int64, N)):
            if t.dtype != dt_ or not t.is_contiguous() or t.shape[0] != n:
                raise _lib.PulseError(f"{name}: expected contiguous {dt_} with {n} rows")
            setattr(g, name, t.data_ptr())
        if fall_root_states.dtype != torch.float32 or fall_root_states.stride(-1) != 1:
            raise _lib.PulseError("fall_root_states must be float32 [P, 13] with contiguous rows")
        if fall_dof_pos.stride() != fall_dof_vel.stride() or fall_dof_pos.dtype != torch.float32 or fall_dof_vel.dtype != torch.float32 \
                or fall_dof_pos.shape[0] != P or fall_dof_vel.shape[0] != P:
            raise _lib.PulseError("fall_dof_pos / fall_dof_vel must be float32 [P, 69] with shared strides")
        g.fall_root_states, g.fall_root_stride = fall_root_states.data_ptr(), fall_root_states.stride(0)
        g.fall_dof_pos, g.fall_dof_vel = fall_dof_pos.data_ptr(), fall_dof_vel.data_ptr()
        g.fall_dof_env_stride, g.fall_dof_elem_stride = fall_dof_pos.stride(0), fall_dof_pos.stride(1)
        g.num_fall_states = P
        g.recovery_prob, g.fall_prob, g.recovery_steps = float(recovery_prob), float(fall_prob), int(recovery_steps)
        for name in ("ref_list", "fall_list", "recovery_list", "class_counts", "env_class", "error", "fall_pick", "fall_key_scratch"):
            setattr(g, name, ws[name].data_ptr())
        with torch.cuda.device(dev):
            _lib.check(self.lib.pulse_reset_getup(self.motion_lib.handle, C.byref(g), N, _lib.current_stream(dev)), "pulse_reset_getup")
        if check:
            self.check_getup_error()
        return ws

    def check_getup_error(self) -> None:
        """Raises PulseError if some fall env of a `reset_getup` call found no free fall state (reads one device word: a host sync)."""
        ws = getattr(self, "_getup_ws", None)
        if ws is not None and int(ws["error"].item()) != 0:
            raise _lib.PulseError(f"reset_getup: {int(ws['error'].item())} fall envs found no free fall state (the reference asserts, "
                                  "humanoid_im_getup.py:172); they took a reference-state episode")

    def getup_amp_init(self, *, body_state: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, amp_obs_buf: torch.Tensor) -> None:
        """`_init_amp_obs` of the fall and recovery envs of the last `reset_getup` (humanoid_amp.py:519-533, humanoid_im_getup.py:190-196),
        run after the simulator's refresh: the current AMP observation into every history row of a fall env, into row 0 of a recovery
        env.  The reference-state envs were back-filled by `reset_getup` itself."""
        ws = getattr(self, "_getup_ws", None)
        if ws is None:
            raise _lib.PulseError("getup_amp_init follows reset_getup")
        a = _lib.GetupAmpArgs()
        a.body_state, a.body_env_stride = _strided(body_state, 13)
        if dof_pos.stride() != dof_vel.stride():
            raise _lib.PulseError("dof_pos and dof_vel must share strides (views of one dof-state tensor)")
        a.dof_pos, a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_pos.data_ptr(), dof_vel.data_ptr(), dof_pos.stride(0), dof_pos.stride(1)
        if not amp_obs_buf.is_contiguous() or amp_obs_buf.shape[-1] != AMP_OBS or amp_obs_buf.shape[0] != ws["env_list"].shape[0]:
            raise _lib.PulseError("amp_obs_buf must be contiguous [N, steps, 196]")
        a.amp_obs_buf, a.num_steps = amp_obs_buf.data_ptr(), int(amp_obs_buf.shape[1])
        a.fall_list, a.recovery_list, a.class_counts = ws["fall_list"].data_ptr(), ws["recovery_list"].data_ptr(), ws["class_counts"].data_ptr()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_getup_amp_init(C.byref(a), int(amp_obs_buf.shape[0]), _lib.current_stream(self.device)), "pulse_getup_amp_init")

    def task_obs(self, *, version: int, body_state: torch.Tensor, progress_buf: torch.Tensor, motion_ids: torch.Tensor,
                 motion_start_times: torch.Tensor, motion_start_offset: torch.Tensor, global_offset: torch.Tensor,
                 track_ids: torch.Tensor, obs_buf: torch.Tensor, time_steps: int = 1, sample_dt: float = 0.0, upright: bool = True,
                 dof_pos: Optional[torch.Tensor] = None, env_ids: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """`HumanoidIm._compute_task_obs` (humanoid_im.py:708-851) for ANY observation version (1, 2, 3, 4/6, 7, 8, 9), tracked-body
        subset and number of future samples (`_fut_tracks`: `time_steps = _num_traj_samples`, `sample_dt = _traj_sample_timestep`,
        :723-729): the MotionLib query of the N * time_steps sample times (one `pulse_motion_state` launch) + one `pulse_im_task_obs`
        launch writing `obs_buf[:, :size]`.  Returns the query (for the `ref_body_*` side buffers, :835-848).
        `track_ids`: int32 device tensor (`_track_bodies_id`).  The fused step kernel remains the path of the default configuration."""
        N = int(body_state.shape[0]) if env_ids is None else int(env_ids.shape[0])
        if env_ids is not None:      # subset call (reset path): gather the rows, the kernel is per env
            body_state, progress_buf, motion_ids = body_state[env_ids], progress_buf[env_ids], motion_ids[env_ids]
            motion_start_times, motion_start_offset, global_offset = motion_start_times[env_ids], motion_start_offset[env_ids], global_offset[env_ids]
            if dof_pos is not None:
                dof_pos = dof_pos[env_ids]
        T = int(time_steps)
        size = int(self.lib.pulse_task_obs_size(int(version), int(track_ids.shape[0]), T))
        if size <= 0:
            raise _lib.PulseError(f"observation version {version} is not built (have 1, 2, 3, 6, 7, 8, 9)")
        if obs_buf.shape[0] != N or obs_buf.shape[1] < size or obs_buf.stride(1) != 1 or obs_buf.dtype != torch.float32:
            raise _lib.PulseError(f"obs_buf must be float32 [{N}, >= {size}] with unit inner stride")
        if track_ids.dtype != torch.int32 or not track_ids.is_contiguous():
            raise _lib.PulseError("track_ids must be a contiguous int32 device tensor")
        if body_state.dim() != 3 or body_state.shape[1] < NUM_BODIES or body_state.shape[2] != 13 or body_state.stride(2) != 1 or body_state.stride(1) != 13:
            raise _lib.PulseError("body_state must be a [N, B>=24, 13] view with row stride 13")
        # motion times of the samples: (progress + 1) * dt + k * sample_dt + start + offset, the reference's operation order (:726 / :732)
        t0 = (progress_buf + 1) * self.cfg.dt
        if T > 1:
            k = torch.arange(T, device=self.device) * sample_dt
            times = (t0[:, None] + k[None, :] + motion_start_times[:, None] + motion_start_offset[:, None]).reshape(-1)
            ids = motion_ids.repeat_interleave(T)
            off = global_offset.repeat_interleave(T, dim=0)
        else:
            times, ids, off = t0 + motion_start_times + motion_start_offset, motion_ids, global_offset
        res = self.motion_lib.get_motion_state(ids, times.to(torch.float32), offset=off.contiguous())
        a = _lib.TaskObsArgs(body_state=body_state.data_ptr(), body_env_stride=body_state.stride(0), track_ids=track_ids.data_ptr(),
                             num_track=int(track_ids.shape[0]), time_steps=T, version=int(version), upright=int(bool(upright)),
                             ref_pos=res["rg_pos"].data_ptr(), ref_rot=res["rb_rot"].data_ptr(), ref_vel=res["body_vel"].data_ptr(),
                             ref_ang_vel=res["body_ang_vel"].data_ptr(), obs=obs_buf.data_ptr(), obs_stride=obs_buf.stride(0), num_envs=N)
        if int(version) == 2:
            if dof_pos is None:
                raise _lib.PulseError("observation version 2 needs dof_pos")
            a.dof_pos, a.dof_env_stride, a.dof_elem_stride, a.ref_dof_pos = dof_pos.data_ptr(), dof_pos.stride(0), dof_pos.stride(1), res["dof_pos"].data_ptr()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_im_task_obs(C.byref(a), _lib.current_stream(self.device)), "pulse_im_task_obs")
        return res

    def fetch_amp_obs_demo(self, num_samples: int) -> torch.Tensor:
        """HumanoidAMP.fetch_amp_obs_demo (humanoid_amp.py:215-230) with HumanoidIm's `_sample_time` = sample_time_interval."""
        ids = self.motion_lib.sample_motions(num_samples)
        return self.build_amp_obs_demo(ids, self.motion_lib.sample_time_interval(ids))


class HumanoidImB200Mixin:
    """Overrides for `phc.env.tasks.humanoid_im.HumanoidIm` (method names and buffer names are the
    reference's).  Usage (see INTEGRATION.md):

        class HumanoidImB200(HumanoidImB200Mixin, HumanoidIm): pass
        phc.utils.parse_task.HumanoidIm = HumanoidImB200      # parse_task.py:67 resolves by name

    `Humanoid.post_physics_step` (humanoid.py:1315-1346) calls, in order, `_compute_reward`,
    `_compute_reset`, `_compute_observations()`.  With cycle_motion off nothing between them mutates
    state, so the first call launches the fused kernel for all three and the other two return.
    """

    _pulse_ready = False

    def _pulse_setup(self):
        self._pulse = HumanoidImCompute.from_task(self)
        self._pulse_motion_lib = self._pulse.motion_lib
        self._pulse_fused_pending = False
        self._pulse_pass_time = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
        unsupported = (getattr(self, "self_obs_v", 1) != 1 or getattr(self, "zero_out_far", False) or getattr(self, "_occl_training", False)
                       or not getattr(self, "_full_body_reward", True) or getattr(self, "add_obs_noise", False))
        obs_v = 6 if int(getattr(self, "obs_v", 6)) == 4 else int(getattr(self, "obs_v", 6))     # obs_v 4 and 6 share a function (:786-787)
        fut = bool(getattr(self, "_fut_tracks", False))
        # the fused step kernel is specialised for the default observation; every other version / tracked-body subset / fut_tracks window
        # goes through the general task-observation kernel (SURVEY 8f-4) with the self observation still taken from the fused kernel
        self._pulse_general_obs = obs_v != 6 or fut or len(self._track_bodies_id) != NUM_BODIES
        if self._pulse_general_obs:
            T = int(getattr(self, "_num_traj_samples", 1)) if fut else 1
            size = int(self._pulse.lib.pulse_task_obs_size(obs_v, len(self._track_bodies_id), T))
            unsupported = unsupported or size <= 0 or (T > 1 and obs_v in (2, 8)) or bool(getattr(self, "_fut_tracks_dropout", False))
            if not unsupported:
                self._pulse_obs_v, self._pulse_T, self._pulse_task_size = obs_v, T, size
                self._pulse_track = self._track_bodies_id.to(self.device, torch.int32).contiguous()
                self._pulse_scratch_obs = torch.zeros(self.num_envs, IM_OBS, device=self.device)
                self._pulse_task_obs = torch.zeros(self.num_envs, size, device=self.device)
        if unsupported:
            raise _lib.PulseError("HumanoidImB200Mixin: unsupported task configuration (needs self_obs_v 1, full-body reward, no zero_out_far / "
                                  "occlusion / observation noise / fut_tracks dropout; obs_v in 1, 2, 3, 4, 6, 7, 8, 9; v2 / v8 without fut_tracks)")
        self._pulse_ready = True

    def resample_motions(self):
        super().resample_motions()
        self._pulse_ready = False  # tables changed: rebuild the packed records lazily

    def _pulse_args(self):
        if not self._pulse_ready:
            self._pulse_setup()
        from .flags_compat import im_eval_mean_reset
        self._pulse.cfg.use_mean_reset = im_eval_mean_reset(self)
        return dict(body_state=self._rigid_body_state_reshaped, dof_vel=self._dof_vel, dof_force=self.dof_force_tensor,
                    progress_buf=self.progress_buf, motion_ids=self._sampled_motion_ids,
                    motion_start_times=self._motion_start_times, motion_start_offset=self._motion_start_times_offset,
                    global_offset=self._global_offset, cycle_counter=self._cycle_counter, obs_buf=self.obs_buf,
                    self_obs_buf=self.self_obs_buf, rew_buf=self.rew_buf, reward_raw=self.reward_raw,
                    reset_buf=self.reset_buf, terminate_buf=self._terminate_buf, pass_time=self._pulse_pass_time,
                    ref_body_pos=self.ref_body_pos, ref_body_vel=self.ref_body_vel, ref_body_rot=self.ref_body_rot,
                    ref_dof_pos=self.ref_dof_pos,
                    # HumanoidImGetup: recovering envs are masked inside the kernel (humanoid_im_getup.py:203-210 never runs behind this mixin)
                    recovery_counter=getattr(self, "_recovery_counter", None))

    def _compute_reward(self, actions):
        args = self._pulse_args()
        if self.cycle_motion:
            self._pulse.step(flags=_lib.STEP_REWARD, **args)
        elif self._pulse_general_obs:      # reward + reset fused; the observation takes the general path in _compute_observations
            self._pulse.step(flags=_lib.STEP_REWARD | _lib.STEP_RESET, **self._pulse_no_obs(args))
            self._pulse_fused_pending = True
        else:
            self._pulse.step(flags=_lib.STEP_ALL, **args)
            self._pulse_fused_pending = True

    @staticmethod
    def _pulse_no_obs(args):
        return {k: v for k, v in args.items() if k not in ("obs_buf", "self_obs_buf", "ref_body_pos", "ref_body_vel", "ref_body_rot", "ref_dof_pos")}

    def _compute_task_obs(self, env_ids=None, save_buffer=True):
        """humanoid_im.py:708-851 for the non-default observation configurations: MotionLib query of the sample times + one
        pulse_im_task_obs launch; returns the [n, task_obs_size] block the reference's _compute_observations concatenates."""
        if not self._pulse_ready:
            self._pulse_setup()
        if not self._pulse_general_obs:
            return super()._compute_task_obs(env_ids, save_buffer)
        n = self.num_envs if env_ids is None else len(env_ids)
        out = self._pulse_task_obs[:n]
        ids = None if env_ids is None else env_ids.to(torch.int64).contiguous()
        res = self._pulse.task_obs(version=self._pulse_obs_v, body_state=self._rigid_body_state_reshaped, progress_buf=self.progress_buf,
                                   motion_ids=self._sampled_motion_ids, motion_start_times=self._motion_start_times,
                                   motion_start_offset=self._motion_start_times_offset, global_offset=self._global_offset,
                                   track_ids=self._pulse_track, obs_buf=out, time_steps=self._pulse_T,
                                   sample_dt=float(getattr(self, "_traj_sample_timestep", 0.0)), upright=bool(getattr(self, "_has_upright_start", True)),
                                   dof_pos=self._dof_pos, env_ids=ids)
        if save_buffer:                    # :835-848 (sample 0 of a fut_tracks window)
            sel = slice(None) if env_ids is None else env_ids
            first = lambda x: x.view(n, self._pulse_T, *x.shape[1:])[:, 0]
            self.ref_body_pos[sel], self.ref_body_vel[sel] = first(res["rg_pos"]), first(res["body_vel"])
            self.ref_body_rot[sel], self.ref_dof_pos[sel] = first(res["rb_rot"]), first(res["dof_pos"])
            if hasattr(self, "ref_body_pos_subset"):
                self.ref_body_pos_subset[sel] = first(res["rg_pos"])[:, self._track_bodies_id]
        return out

    def _compute_reset(self):
        if self._pulse_fused_pending:
            return
        # cycle_motion: wrapped envs get a new start time / offset before the reset + obs queries
        # (humanoid_im.py:1125-1146); this host-side block keeps the reference's ops (and its syncs).
        wrapped = self._pulse_pass_time.bool()
        if wrapped.any():
            self._motion_start_times_offset[wrapped] = -self.progress_buf[wrapped] * self.dt
            self._motion_start_times[wrapped] = self._sample_time(self._sampled_motion_ids[wrapped])
            self._cycle_counter[wrapped] = 60
            root = self._pulse_motion_lib.get_root_pos_smpl(self._sampled_motion_ids[wrapped], self._motion_start_times[wrapped])
            self._global_offset[wrapped, :2] = self._humanoid_root_states[wrapped, :2] - root["root_pos"][:, :2]
        self._pulse.step(flags=_lib.STEP_RESET | _lib.STEP_OBS, **self._pulse_args())
        self._pulse_fused_pending = True

    def _compute_observations(self, env_ids=None):
        if getattr(self, "_pulse_general_obs", False) or not self._pulse_ready:
            args = self._pulse_args()
            if self._pulse_general_obs:
                # humanoid_im.py:677-706: obs = [self obs (fused kernel, observation mode, into a scratch row) | task obs (general kernel)]
                self._pulse_fused_pending = False
                if env_ids is not None and len(env_ids) == 0:
                    return
                a = self._pulse_no_obs(args)
                if env_ids is not None:
                    a["env_ids"] = env_ids.to(torch.int64).contiguous()
                self._pulse.step(flags=_lib.STEP_OBS, obs_buf=self._pulse_scratch_obs, self_obs_buf=self.self_obs_buf, **a)
                task = self._compute_task_obs(env_ids)
                sel = slice(None) if env_ids is None else env_ids
                self.obs_buf[sel, :SELF_OBS] = self.self_obs_buf[sel]
                self.obs_buf[sel, SELF_OBS:SELF_OBS + task.shape[1]] = task
                return
        if env_ids is None and self._pulse_fused_pending:
            self._pulse_fused_pending = False
            return
        self._pulse_fused_pending = False
        args = self._pulse_args()
        if env_ids is not None:
            if len(env_ids) == 0:
                return
            args["env_ids"] = env_ids.to(torch.int64).contiguous()
        self._pulse.step(flags=_lib.STEP_OBS, **args)

    def _reset_envs(self, env_ids):
        """Humanoid._reset_envs + HumanoidAMP._reset_envs (humanoid.py:574-587, humanoid_amp.py:347-356) for the reference-state
        initialisations (`StateInit.Random` / `Start`): `_reset_actors` -> `_reset_ref_state_init` -> `_sample_ref_state` ->
        `_set_env_state` (humanoid_im.py:921-989, humanoid_amp.py:468-488, :565-597) and `_init_amp_obs` (:519-563) are ONE
        `pulse_reset_ref_state` launch writing the simulator views and `_amp_obs_buf` in place.  What stays the reference's: the
        start-time draws come from `torch.rand(env_ids.shape)` exactly as `sample_time_interval` makes them (motion_lib_base.py:411-420:
        the process RNG stream is consumed identically), `_reset_env_tensors` (the gym indexed setters, humanoid.py:589-609),
        `_refresh_sim_tensors` with its `_reset_rb_*` restore (humanoid_amp.py:598-620) and `_compute_observations(env_ids)`.
        Default / Hybrid state initialisation is handed back to the reference."""
        name = getattr(getattr(self, "_state_init", None), "name", None)
        # HumanoidImGetup splits the reset envs into recovery / fall-state / reference-state episodes inside its own `_reset_actors`
        # (humanoid_im_getup.py:135-182): HumanoidImGetupB200Mixin below serves it; behind this mixin alone it stays the reference's.
        if len(env_ids) == 0 or name not in ("Random", "Start") or hasattr(self, "_recovery_counter"):
            return super()._reset_envs(env_ids)
        if not self._pulse_ready:
            self._pulse_setup()
        env_ids = env_ids.to(torch.int64).contiguous()
        self._reset_default_env_ids = []
        self._state_reset_happened = True
        self._pulse_draw_phase(env_ids, name)
        self._pulse.reset_envs(env_ids=env_ids, phase=self._pulse_phase, motion_ids=self._sampled_motion_ids,
                               motion_start_times=self._motion_start_times, motion_start_offset=self._motion_start_times_offset,
                               global_offset=self._global_offset, progress_buf=self.progress_buf, cycle_counter=self._cycle_counter,
                               terminate_buf=self._terminate_buf, root_states=self._humanoid_root_states, dof_pos=self._dof_pos,
                               dof_vel=self._dof_vel, rigid_body_state=self._rigid_body_state_reshaped,
                               contact_forces=self._contact_forces, amp_obs_buf=self._amp_obs_buf)
        self._reset_ref_env_ids = env_ids
        self._reset_ref_motion_ids = self._sampled_motion_ids[env_ids]
        self._reset_ref_motion_times = self._motion_start_times[env_ids]
        # gym's refresh rewrites the rigid-body tensor from the simulator: the reference keeps clones and restores them after it
        self._reset_rb_pos, self._reset_rb_rot = self._rigid_body_pos[env_ids].clone(), self._rigid_body_rot[env_ids].clone()
        self._reset_rb_vel, self._reset_rb_ang_vel = self._rigid_body_vel[env_ids].clone(), self._rigid_body_ang_vel[env_ids].clone()
        self._reset_env_tensors(env_ids)
        self._refresh_sim_tensors()
        self._compute_observations(env_ids)
        # _init_amp_obs: rows 0 .. steps-1 of `_amp_obs_buf[env_ids]` were written by the launch above (row 0 from the state just set)

    def _pulse_draw_phase(self, env_ids, name):
        from .flags_compat import flags_test
        if getattr(self, "_pulse_phase", None) is None or self._pulse_phase.shape[0] != self.num_envs:
            self._pulse_phase = torch.zeros(self.num_envs, device=self.device)
        if name == "Start" or flags_test():                    # motion_times = 0 (humanoid_im.py:971-977)
            self._pulse_phase.zero_()
        else:
            self._pulse_phase[env_ids] = torch.rand(env_ids.shape, device=self.device)

    def _pulse_amp_fused(self, env_ids) -> bool:
        """The fused AMP launch (history shift + current observation) covers the whole-batch call of the default configuration; one
        predicate for BOTH overrides below, so the shift is skipped exactly when the fused launch performs it."""
        return env_ids is None and getattr(self, "amp_obs_v", 1) == 1 and bool(getattr(self, "_has_dof_subset", True))

    def _update_hist_amp_obs(self, env_ids=None):
        if self._pulse_amp_fused(env_ids):
            return  # folded into _compute_amp_observations (one launch does shift + write)
        super()._update_hist_amp_obs(env_ids)

    def _compute_amp_observations(self, env_ids=None):
        if not self._pulse_amp_fused(env_ids):
            return super()._compute_amp_observations(env_ids)
        if not self._pulse_ready:
            self._pulse_setup()
        self._pulse.amp_obs(body_state=self._rigid_body_state_reshaped, dof_pos=self._dof_pos, dof_vel=self._dof_vel,
                            amp_obs_buf=self._amp_obs_buf, shift_history=True)

class HumanoidImGetupB200Mixin(HumanoidImB200Mixin):
    """`HumanoidImB200Mixin` for `phc.env.tasks.humanoid_im_getup.HumanoidImGetup` (PULSE's distillation task, env_im_vae.yaml),
    whose reset it also serves (see INTEGRATION.md):

        class HumanoidImGetupB200(HumanoidImGetupB200Mixin, HumanoidImGetup): pass

    The step path is the base mixin's (recovering envs are masked inside the fused kernel through `_recovery_counter`)."""

    def _reset_envs(self, env_ids):
        """HumanoidImGetup._reset_envs (humanoid_im_getup.py:135-196 over humanoid.py:574-609, humanoid_amp.py:347-356, :519-620) with
        `pulse_reset_getup` in place of `_reset_actors`.  After the start-time draws, the recovery / fall draws of env_ids come from
        `torch.rand((2, n))` and one key per fall state from `torch.rand(P)`, so `torch.manual_seed` fixes them.  The reference's
        `_reset_env_tensors` and `_refresh_sim_tensors` follow; what would sync on a data-dependent list is replaced: the `_reset_rb_*`
        restore covers all of env_ids and keeps the saved rows where the env took a reference-state episode (a device mask), and
        `_init_amp_obs` of the fall / recovery envs is `getup_amp_init`.  `_generate_fall_states`, `update_getup_schedule` and
        `_update_recovery_count` stay the reference's."""
        name = getattr(getattr(self, "_state_init", None), "name", None)
        if len(env_ids) == 0 or name not in ("Random", "Start"):
            return super()._reset_envs(env_ids)
        if not self._pulse_ready:
            self._pulse_setup()
        env_ids = env_ids.to(torch.int64).contiguous()
        self._reset_default_env_ids = []
        self._pulse_draw_phase(env_ids, name)
        n, dev = env_ids.shape[0], self.device
        if getattr(self, "_pulse_getup_u", None) is None or self._pulse_getup_u.shape[1] != self.num_envs:
            self._pulse_getup_u = torch.ones(2, self.num_envs, device=dev)
        self._pulse_getup_u[:, env_ids] = torch.rand((2, n), device=dev)
        keys = torch.rand(self._fall_root_states.shape[0], device=dev)
        ws = self._pulse.reset_getup(
            env_ids=env_ids, phase=self._pulse_phase, recovery_u=self._pulse_getup_u[0], fall_u=self._pulse_getup_u[1], fall_keys=keys,
            motion_ids=self._sampled_motion_ids, motion_start_times=self._motion_start_times, motion_start_offset=self._motion_start_times_offset,
            global_offset=self._global_offset, progress_buf=self.progress_buf, cycle_counter=self._cycle_counter, terminate_buf=self._terminate_buf,
            root_states=self._humanoid_root_states, dof_pos=self._dof_pos, dof_vel=self._dof_vel, rigid_body_state=self._rigid_body_state_reshaped,
            contact_forces=self._contact_forces, amp_obs_buf=self._amp_obs_buf, recovery_counter=self._recovery_counter,
            available_fall_states=self.availalbe_fall_states, fall_id_assignments=self.fall_id_assignments,
            fall_root_states=self._fall_root_states, fall_dof_pos=self._fall_dof_pos, fall_dof_vel=self._fall_dof_vel,
            recovery_prob=float(self._recovery_episode_prob), fall_prob=float(self._fall_init_prob), recovery_steps=int(self._recovery_steps))
        self._reset_fall_env_ids = []                          # _init_amp_obs_default runs below, not through the reference
        saved = [v[env_ids].clone() for v in (self._rigid_body_pos, self._rigid_body_rot, self._rigid_body_vel, self._rigid_body_ang_vel)]
        self._state_reset_happened = False                     # the reference's list-indexed restore is the masked one below
        self._reset_env_tensors(env_ids)
        self._refresh_sim_tensors()
        is_ref = (ws["env_class"][env_ids] == _lib.GETUP_REF).view(-1, 1, 1)
        for v, s in zip((self._rigid_body_pos, self._rigid_body_rot, self._rigid_body_vel, self._rigid_body_ang_vel), saved):
            v[env_ids] = torch.where(is_ref, s, v[env_ids])
        self._compute_observations(env_ids)
        self._pulse.getup_amp_init(body_state=self._rigid_body_state_reshaped, dof_pos=self._dof_pos, dof_vel=self._dof_vel,
                                   amp_obs_buf=self._amp_obs_buf)
