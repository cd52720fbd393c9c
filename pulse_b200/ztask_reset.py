"""Reference-state reset of the latent-space tasks HumanoidReach(Z) / HumanoidSpeed(Z) / HumanoidStrike(Z) on the device
(`pulse_reset_ztask`, `pulse_ztask_reset_task`): `HumanoidAMPTask._reset_envs` for StateInit.Random / Start and the SMPL humanoid,
without the reference's SMPL mesh forward and its host synchronisations.

The reference lifts every reset pose onto the ground with a full SMPL forward (`_get_fixed_smpl_state_from_motionlib`,
humanoid_amp.py:382-430).  For one body shape the lift of frame f is `floor(f) + root_z - 0.02`, with floor(f) = min_v V_z - J0_z of
frame f's pose at zero translation, so the device takes `floor` as a per-frame table: `smpl_ground_table` builds it once with the
task's own parser.

Call order of one reset, as in the reference: `reset_envs` (state, counters, strike target, AMP history), the simulator's refresh, the
task observation of the reset envs, then `reset_task` (the reach target / target speed).  Draws are injected per env (tests; a caller
that wants the reference's own random stream) or made by Philox4x32-10 inside the kernels (word layout: include/pulse_b200.h).
"""
import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from .motion_lib import MotionLibB200

AMP_WIDTHS = (196, 195)
SMPLX_AMP_WIDTHS = (_lib.SMPLX_AMP_OBS, _lib.SMPLX_AMP_OBS_NO_HEIGHT)
_POSE = {"reach": _lib.ZPOSE_ROOT_XY_ZERO, "strike": _lib.ZPOSE_ROOT_XY_ZERO, "speed": _lib.ZPOSE_FACE_X}
_INIT = {"Random": _lib.ZINIT_RANDOM, "Start": _lib.ZINIT_START}


def smpl_ground_table(motion_aa: torch.Tensor, parser, betas: torch.Tensor, chunk: int = 4096) -> torch.Tensor:
    """floor[f] = min over vertices of V_z - J0_z for frame f's pose `motion_aa[f]` and the shape `betas` at zero translation:
    `parser.get_joints_verts(pose, betas, trans)` -> (vertices [B,V,3], joints [B,J,3]) is the task's SMPL parser.  fp32 [F] on the
    device of `motion_aa`."""
    F = int(motion_aa.shape[0])
    out = torch.empty(F, dtype=torch.float32, device=motion_aa.device)
    b = betas.reshape(1, -1).to(motion_aa.device)
    with torch.no_grad():
        for s in range(0, F, chunk):
            pose = motion_aa[s:s + chunk]
            n = int(pose.shape[0])
            verts, joints = parser.get_joints_verts(pose, b.expand(n, -1), torch.zeros(n, 3, dtype=pose.dtype, device=pose.device))
            out[s:s + n] = verts[..., 2].min(dim=-1).values - joints[:, 0, 2]
    return out


def _f32(t: torch.Tensor, rows: int, name: str, cols: Optional[int] = None):
    ok = t.dtype == torch.float32 and t.is_contiguous() and t.shape[0] == rows and (cols is None or (t.dim() == 2 and t.shape[1] == cols))
    if not ok:
        raise _lib.PulseError(f"{name} must be contiguous float32 [{rows}{', %d' % cols if cols else ''}]")
    return t.data_ptr()


class ZTaskResetB200:
    """The reset of one latent-space task over N envs.  kind: "reach" / "speed" / "strike"; `floor` the per-frame table of
    `smpl_ground_table` (at least the MotionLib's frame count); `upright` = _has_upright_start; `amp_root_height_obs` chooses the
    196- or 195-float AMP rows (ampRootHeightObs, False in env_pulse_amp.yaml).

    A 52-body MotionLib (SMPL-X, PULSE-X) serves the speed task through `pulse_reset_ztask_smplx`: views of >= 52 bodies and 153 dofs,
    `upright` False as in env_pulsex_amp.yaml (True is refused: the SMPL-X step takes the non-upright heading), and the AMP history
    in the SMPL-X rows: 466 floats, or 465 without the root height (`amp_root_height_obs`).  SMPL-X reach and strike go through the
    subclass SmplxTargetResetB200."""
    # the tasks a 52-body MotionLib serves here, and their entry point (SmplxTargetResetB200 sets both)
    smplx_kinds, smplx_entry = ("speed",), "pulse_reset_ztask_smplx"

    def __init__(self, kind: str, motion_lib: MotionLibB200, floor: torch.Tensor, *, upright: bool = True, state_init: str = "Random",
                 amp_root_height_obs: bool = False, dt: float = float(torch.tensor(1.0 / 60.0, dtype=torch.float32) * 2),
                 near_prob: float = 0.5, near_dist: float = 1.5, tar_dist_min: float = 0.5, tar_dist_max: float = 10.0,
                 reach_dist_max: float = 1.0, tar_height_min: float = 0.5, tar_height_max: float = 1.5,
                 tar_speed_min: float = 0.0, tar_speed_max: float = 5.0, change_steps_min: int = 100, change_steps_max: int = 200):
        if kind not in _POSE:
            raise _lib.PulseError(f"unknown latent task {kind!r} (reach, speed, strike)")
        if state_init not in _INIT:
            raise _lib.PulseError(f"state_init {state_init!r}: the device reset serves Random and Start")
        self.kind, self.motion_lib, self.device = kind, motion_lib, motion_lib._device
        self.smplx = bool(getattr(motion_lib, "smplx", False))
        if self.smplx and kind not in self.smplx_kinds:
            raise _lib.PulseError(f"the SMPL-X {type(self).__name__} serves {' and '.join(self.smplx_kinds)}, not {kind!r}")
        if self.smplx and upright:
            raise _lib.PulseError("the SMPL-X reset takes upright=False (env_pulsex_amp.yaml: has_upright_start False), the heading its "
                                  "step kernel uses")
        self.bodies, self.dofs = (_lib.SMPLX_BODIES, _lib.SMPLX_DOF) if self.smplx else (24, 69)
        self.pose_mode, self.init_code = _POSE[kind], _INIT[state_init]
        if floor.dtype != torch.float32 or floor.dim() != 1 or floor.device != self.device:
            raise _lib.PulseError("floor must be a float32 [F] table on the MotionLib's device")
        if floor.shape[0] < motion_lib.gts.shape[0]:
            raise _lib.PulseError(f"floor table has {floor.shape[0]} frames, the MotionLib {motion_lib.gts.shape[0]}")
        self.floor = floor.contiguous()
        self.upright, self.state_init, self.dt = bool(upright), state_init, float(dt)
        self.amp_width = (SMPLX_AMP_WIDTHS if self.smplx else AMP_WIDTHS)[0 if amp_root_height_obs else 1]
        self.strike = (float(near_prob), float(near_dist), float(tar_dist_min), float(tar_dist_max))
        self.reach = (float(reach_dist_max), float(tar_height_min), float(tar_height_max))
        self.speed = (float(tar_speed_min), float(tar_speed_max))
        self.change_steps = (int(change_steps_min), int(change_steps_max))
        self.lib = _lib.load()
        self._ws = None

    def _workspace(self, N: int) -> Dict[str, torch.Tensor]:
        if self._ws is None or self._ws["env_list"].shape[0] != N:
            dev = self.device
            self._ws = {"env_list": torch.zeros(N, dtype=torch.int64, device=dev), "actor_list": torch.zeros(N, dtype=torch.int32, device=dev),
                        "tar_actor_list": torch.zeros(N, dtype=torch.int32, device=dev), "count": torch.zeros(1, dtype=torch.int32, device=dev)}
        return self._ws

    def reset_envs(self, *, root_states: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, rigid_body_state: torch.Tensor,
                   progress_buf: torch.Tensor, sampled_motion_ids: torch.Tensor, motion_start_times: torch.Tensor,
                   reset_buf: Optional[torch.Tensor] = None, env_ids: Optional[torch.Tensor] = None, terminate_buf: Optional[torch.Tensor] = None,
                   contact_forces: Optional[torch.Tensor] = None, amp_obs_buf: Optional[torch.Tensor] = None,
                   actor_ids: Optional[torch.Tensor] = None, target_states: Optional[torch.Tensor] = None,
                   tar_actor_ids: Optional[torch.Tensor] = None, motion_ids: Optional[torch.Tensor] = None,
                   motion_u: Optional[torch.Tensor] = None, phase: Optional[torch.Tensor] = None,
                   strike_u: Optional[torch.Tensor] = None, seed: int = 0, offset: int = 0,
                   offset_dev: Optional[torch.Tensor] = None, amp_fresh: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """`pulse_reset_ztask` for the envs of `reset_buf` (mask) or `env_ids` (int64 list): clip and start time, ground fix, the task's
        pose adjustment, the simulator views written in place, `_sampled_motion_ids` / `_motion_start_times`, counters and contact forces
        cleared, the strike target (kind "strike": `target_states` is the [N, 13] view of the target actors) and the AMP history
        [N, steps, 195 | 196].  `env_ids` must be ascending (what `nonzero` returns): an id out of range or not above its predecessor
        is skipped.  Injected draws are per ENV: `motion_ids` int64 [N] (the clips themselves) or `motion_u` [N] (uniforms turned into
        clips through the sampling CDF), `phase` [N], `strike_u` [N, 4]; None -> Philox on (seed, env, offset [+ *offset_dev]).  `amp_fresh`
        int32 [N] (with amp_obs_buf): set to 1 for every reset env, for `pulse_amp_obs_row`.  Returns the workspace {'env_list', 'actor_list', 'tar_actor_list', 'count'} (device)."""
        a, ws = self._args(root_states=root_states, dof_pos=dof_pos, dof_vel=dof_vel, rigid_body_state=rigid_body_state, progress_buf=progress_buf,
                           sampled_motion_ids=sampled_motion_ids, motion_start_times=motion_start_times, reset_buf=reset_buf, env_ids=env_ids,
                           terminate_buf=terminate_buf, contact_forces=contact_forces, amp_obs_buf=amp_obs_buf, actor_ids=actor_ids,
                           target_states=target_states, tar_actor_ids=tar_actor_ids, motion_ids=motion_ids, motion_u=motion_u, phase=phase,
                           strike_u=strike_u, seed=seed, offset=offset, offset_dev=offset_dev, amp_fresh=amp_fresh)
        fn, handle = (self.smplx_entry, self.motion_lib.smplx_handle) if self.smplx else ("pulse_reset_ztask", self.motion_lib.handle)
        with torch.cuda.device(self.device):
            _lib.check(getattr(self.lib, fn)(handle, C.byref(a), int(progress_buf.shape[0]), _lib.current_stream(self.device)), fn)
        return ws

    def _args(self, *, root_states, dof_pos, dof_vel, rigid_body_state, progress_buf, sampled_motion_ids, motion_start_times, reset_buf, env_ids,
              terminate_buf, contact_forces, amp_obs_buf, actor_ids, target_states, tar_actor_ids, motion_ids, motion_u, phase, strike_u, seed,
              offset, offset_dev, amp_fresh=None):
        """The checked `pulse_ztask_reset_args_t` of a `reset_envs` call, and the workspace it writes."""
        N = int(progress_buf.shape[0])
        dev = self.device
        if (reset_buf is None) == (env_ids is None):
            raise _lib.PulseError("reset_envs takes either the reset_buf mask or an explicit env_ids list")

        def view(t, name, dtype, shape_ok, layout_ok, what):
            if t.dtype != dtype or t.device != dev or t.shape[0] != N or not shape_ok or not layout_ok:
                raise _lib.PulseError(f"{name} must be a {dtype} view on {dev} with {N} rows, {what}")

        B, D = self.bodies, self.dofs
        view(rigid_body_state, "rigid_body_state", torch.float32, rigid_body_state.dim() == 3 and rigid_body_state.shape[1] >= B,
             rigid_body_state.stride(1) == 13 and rigid_body_state.stride(2) == 1, f"[N, B >= {B}, 13] with row stride 13")
        view(root_states, "root_states", torch.float32, root_states.dim() == 2 and root_states.shape[1] >= 13, root_states.stride(1) == 1,
             "[N, >= 13] with contiguous rows")
        for name, t in (("dof_pos", dof_pos), ("dof_vel", dof_vel)):
            view(t, name, torch.float32, t.dim() == 2 and t.shape[1] == D, t.stride() == dof_pos.stride(), f"[N, {D}], dof_pos and dof_vel sharing strides")
        if terminate_buf is not None:
            view(terminate_buf, "terminate_buf", torch.int64, terminate_buf.dim() == 1, terminate_buf.is_contiguous(), "contiguous [N]")
        if contact_forces is not None:
            view(contact_forces, "contact_forces", torch.float32, contact_forces.dim() == 3 and contact_forces.shape[2] == 3,
                 contact_forces.stride(1) == 3 and contact_forces.stride(2) == 1, "[N, B, 3] with contiguous bodies")
        if (self.kind == "strike") != (target_states is not None):
            raise _lib.PulseError("target_states is required by the strike task and only by it")
        if target_states is not None:
            view(target_states, "target_states", torch.float32, target_states.dim() == 2 and target_states.shape[1] >= 13,
                 target_states.stride(1) == 1, "[N, >= 13] with contiguous rows")
        ws = self._workspace(N)
        a = _lib.ZTaskResetArgs()
        if reset_buf is not None:
            if reset_buf.dtype != torch.int64 or reset_buf.shape[0] != N or not reset_buf.is_contiguous() or reset_buf.device != dev:
                raise _lib.PulseError("reset_buf must be int64 [N]")
            a.reset_buf = reset_buf.data_ptr()
        else:
            if env_ids.dtype != torch.int64 or not env_ids.is_contiguous() or env_ids.device != dev or env_ids.dim() != 1 or env_ids.shape[0] > N:
                raise _lib.PulseError(f"env_ids must be a contiguous int64 list of at most {N} ascending ids on {dev}")
            a.env_ids_in, a.num_ids = (env_ids.data_ptr() if env_ids.numel() else ws["env_list"].data_ptr()), int(env_ids.shape[0])
        if motion_ids is not None:
            if motion_ids.dtype != torch.int64 or not motion_ids.is_contiguous() or motion_ids.shape[0] != N:
                raise _lib.PulseError("motion_ids must be contiguous int64 [N] (one clip per env)")
            a.motion_ids_in = motion_ids.data_ptr()
        else:
            a.sampling_cdf = self.motion_lib.sampling_cdf().data_ptr()
            if motion_u is not None:
                a.motion_u = _f32(motion_u, N, "motion_u")
        if phase is not None:
            a.phase = _f32(phase, N, "phase")
        if strike_u is not None:
            a.strike_u = _f32(strike_u, N, "strike_u", 4)
        a.seed, a.offset = int(seed) & (2 ** 64 - 1), int(offset) & (2 ** 64 - 1)
        if offset_dev is not None:
            a.offset_dev = offset_dev.data_ptr()
        a.floor, a.floor_len = self.floor.data_ptr(), int(self.floor.shape[0])
        a.pose_mode, a.upright, a.state_init, a.dt = self.pose_mode, int(self.upright), self.init_code, self.dt
        if amp_obs_buf is not None:
            if not amp_obs_buf.is_contiguous() or amp_obs_buf.dim() != 3 or amp_obs_buf.shape[0] != N or amp_obs_buf.shape[-1] != self.amp_width:
                raise _lib.PulseError(f"amp_obs_buf must be contiguous [N, steps, {self.amp_width}] (the reset's AMP rows)")
            if amp_obs_buf.dtype != torch.float32 or amp_obs_buf.device != dev:
                raise _lib.PulseError(f"amp_obs_buf must be float32 on {dev}")
            a.amp_obs_buf, a.num_amp_steps, a.amp_width = amp_obs_buf.data_ptr(), int(amp_obs_buf.shape[1]), self.amp_width
        if amp_fresh is not None:
            if amp_obs_buf is None or amp_fresh.dtype != torch.int32 or amp_fresh.shape != (N,) or not amp_fresh.is_contiguous() or amp_fresh.device != dev:
                raise _lib.PulseError(f"amp_fresh must be contiguous int32 [{N}] on {dev}, given with amp_obs_buf")
            a.amp_fresh = amp_fresh.data_ptr()
        for name, t, dt_ in (("sampled_motion_ids", sampled_motion_ids, torch.int64), ("motion_start_times", motion_start_times, torch.float32),
                             ("progress_buf", progress_buf, torch.int64)):
            if t.dtype != dt_ or not t.is_contiguous() or t.shape[0] != N or t.device != dev:
                raise _lib.PulseError(f"{name}: expected contiguous {dt_} with {N} rows on {dev}")
            setattr(a, name, t.data_ptr())
        if terminate_buf is not None:
            a.terminate_buf = terminate_buf.data_ptr()
        a.root_states, a.root_env_stride = root_states.data_ptr(), root_states.stride(0)
        a.dof_pos, a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_pos.data_ptr(), dof_vel.data_ptr(), dof_pos.stride(0), dof_pos.stride(1)
        a.rigid_body_state, a.body_env_stride = rigid_body_state.data_ptr(), rigid_body_state.stride(0)
        if contact_forces is not None:
            a.contact_forces, a.contact_env_stride, a.contact_bodies = contact_forces.data_ptr(), contact_forces.stride(0), int(contact_forces.shape[1])
        if target_states is not None:
            if target_states.stride(-1) != 1 or target_states.shape[-1] < 13:
                raise _lib.PulseError("target_states must be an [N, 13] view with contiguous rows")
            a.target_states, a.target_env_stride = target_states.data_ptr(), target_states.stride(0)
            a.near_prob, a.near_dist, a.tar_dist_min, a.tar_dist_max = self.strike
        for name, t in (("actor_ids", actor_ids), ("tar_actor_ids", tar_actor_ids)):
            if t is not None:
                if t.dtype != torch.int32 or t.shape[0] != N or not t.is_contiguous() or t.device != dev:
                    raise _lib.PulseError(f"{name} must be contiguous int32 [N] on {dev}")
                setattr(a, name, t.data_ptr())
        a.env_list, a.actor_list, a.count = ws["env_list"].data_ptr(), ws["actor_list"].data_ptr(), ws["count"].data_ptr()
        if self.kind == "strike":
            a.tar_actor_list = ws["tar_actor_list"].data_ptr()
        return a, ws

    def observe(self, task, rigid_body_state: torch.Tensor, progress_buf: torch.Tensor, **kw) -> None:
        """_compute_observations(env_ids) of the envs of the last `reset_envs`, run after the simulator's refresh: `task` is the
        ReachTaskB200 / SpeedTaskB200 / StrikeTaskB200 whose observation rows to write (`pulse_reach_obs_list` / `pulse_ztask_obs_list`
        over the device-side list); `kw` are its `observe_list` arguments (strike: `target_states`)."""
        if self._ws is None:
            raise _lib.PulseError("observe follows reset_envs")
        task.observe_list(rigid_body_state, self._ws["env_list"], self._ws["count"], progress_buf, **kw)

    def reset_task(self, *, progress_buf: torch.Tensor, change_steps: torch.Tensor, tar_pos: Optional[torch.Tensor] = None,
                   tar_speed: Optional[torch.Tensor] = None, rand: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None,
                   seed: int = 0, offset: int = 0, offset_dev: Optional[torch.Tensor] = None) -> None:
        """`_reset_task` of the reach (`tar_pos` [N, 3]) or speed (`tar_speed` [N]) task over the envs of the last `reset_envs`, run after
        their observation.  `change_steps` is `_tar_change_steps` / `_speed_change_steps`.  Injected draws per ENV: `rand` [N, 3] (reach)
        or [N] (speed) uniforms, `steps` int64 [N] randint results; None -> Philox."""
        if self.kind == "strike":
            raise _lib.PulseError("the strike task has no _reset_task")
        if self._ws is None:
            raise _lib.PulseError("reset_task follows reset_envs")
        N = int(progress_buf.shape[0])
        t = _lib.ZTaskTaskArgs()
        t.env_list, t.count = self._ws["env_list"].data_ptr(), self._ws["count"].data_ptr()
        for name, x, dt_ in (("progress_buf", progress_buf, torch.int64), ("change_steps", change_steps, torch.int64)):
            if x.dtype != dt_ or not x.is_contiguous() or x.shape[0] != N:
                raise _lib.PulseError(f"{name}: expected contiguous {dt_} with {N} rows")
            setattr(t, name, x.data_ptr())
        if self.kind == "reach":
            t.kind = _lib.ZTASK_REACH
            if tar_pos is None:
                raise _lib.PulseError("the reach task needs tar_pos")
            t.tar_pos = _f32(tar_pos, N, "tar_pos", 3)
            if rand is not None:
                t.rand = _f32(rand, N, "rand", 3)
            dmax, hmin, hmax = self.reach
            t.dist_max, t.height_scale, t.height_min = dmax, hmax - hmin, hmin
        else:
            t.kind = _lib.ZTASK_SPEED
            if tar_speed is None:
                raise _lib.PulseError("the speed task needs tar_speed")
            t.tar_speed = _f32(tar_speed, N, "tar_speed")
            if rand is not None:
                t.rand = _f32(rand, N, "rand")
            smin, smax = self.speed
            t.speed_scale, t.speed_min = smax - smin, smin
        if steps is not None:
            if steps.dtype != torch.int64 or not steps.is_contiguous() or steps.shape[0] != N:
                raise _lib.PulseError("steps must be contiguous int64 [N]")
            t.steps_in = steps.data_ptr()
        t.steps_min, t.steps_max = self.change_steps
        t.seed, t.offset = int(seed) & (2 ** 64 - 1), int(offset) & (2 ** 64 - 1)
        if offset_dev is not None:
            t.offset_dev = offset_dev.data_ptr()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_ztask_reset_task(C.byref(t), N, _lib.current_stream(self.device)), "pulse_ztask_reset_task")


class SmplxTargetResetB200(ZTaskResetB200):
    """The reset of the SMPL-X reach and strike tasks (PULSE-X) over a 52-body MotionLib, through `pulse_reset_smplx_target`: the
    reference-state reset of ZTaskResetB200 with the root's xy zeroed (humanoid_reach.py:46-48, humanoid_strike.py:147-150), the strike
    target placed around it (`target_states`), the AMP back-fill in the SMPL-X rows, and reach's `reset_task`.  `upright=True` is
    refused.  It is a subclass rather than a wider ZTaskResetB200 so that ZTaskResetB200 keeps its contract: over SMPL-X tables it
    serves the speed task and refuses the others."""
    smplx_kinds, smplx_entry = ("reach", "strike"), "pulse_reset_smplx_target"

    def __init__(self, kind: str, motion_lib: MotionLibB200, floor: torch.Tensor, **kw):
        if not getattr(motion_lib, "smplx", False):
            raise _lib.PulseError("SmplxTargetResetB200 takes a 52-body (SMPL-X) MotionLib; ZTaskResetB200 serves the SMPL one")
        super().__init__(kind, motion_lib, floor, **kw)


_KEY_BODY_IDS = (7, 3, 22, 17)                                                     # env_im.yaml / env_pulse_amp.yaml key bodies
_DOF_SUBSET = tuple(k for k in range(69) if (k // 3) not in (3, 7, 17, 22))        # humanoid.py:397,417-421


# SMPL-X (smplx_humanoid.yaml, env_pulsex_amp.yaml): R_Ankle, L_Ankle, R_Wrist, L_Wrist in SMPLH_MUJOCO_NAMES order, and the dofs of
# joints 0..50 without L_Toe (3) and R_Toe (7) (humanoid.py:404-421): 147 of 153
SMPLX_KEY_BODY_IDS = (7, 3, 36, 17)
SMPLX_DOF_SUBSET = tuple(k for k in range(153) if (k // 3) not in (3, 7))


def check_amp_layout(task, who: str, smplx: bool = False) -> None:
    """Refuses, naming the option, a task whose AMP observation the device rows do not build: amp_obs_v other than 1, other key bodies
    (_key_body_ids) or another dof_subset than the layout's (SMPL: `_KEY_BODY_IDS` / `_DOF_SUBSET`; SMPL-X: `SMPLX_KEY_BODY_IDS` /
    `SMPLX_DOF_SUBSET`).  A PULSE-X integration calls it with smplx=True on its HumanoidSpeedZ task before wiring the AMP part."""
    keys, subset, dropped = (SMPLX_KEY_BODY_IDS, SMPLX_DOF_SUBSET, "toes") if smplx else (_KEY_BODY_IDS, _DOF_SUBSET, "toes and hands")
    if int(getattr(task, "amp_obs_v", 1)) != 1:
        raise _lib.PulseError(f"{who}: amp_obs_v {task.amp_obs_v}, the device AMP rows are amp_obs_v 1")
    if tuple(int(i) for i in task._key_body_ids.tolist()) != keys:
        raise _lib.PulseError(f"{who}: keyBodies (_key_body_ids) other than R_Ankle, L_Ankle, R_Wrist, L_Wrist {keys}")
    if not getattr(task, "_has_dof_subset", False) or tuple(int(i) for i in task.dof_subset.tolist()) != subset:
        raise _lib.PulseError(f"{who}: a dof_subset (_has_dof_subset) other than the one without {dropped}")


def smpl_reset_tables(task, ml, who: str):
    """The checks shared by the device resets' mixins and what they build once per MotionLib load: the task's MotionLib as a
    `MotionLibB200` and the floor table of its one body shape.  Refuses, naming the option, what the device reset does not serve."""
    if getattr(task, "humanoid_type", None) != "smpl":
        raise _lib.PulseError(f"{who}: humanoid_type {getattr(task, 'humanoid_type', None)!r}, the device reset serves 'smpl'")
    check_amp_layout(task, who)
    shapes = task.humanoid_shapes
    if bool((shapes != shapes[0:1]).any()):              # once per MotionLib load: one host read
        raise _lib.PulseError(f"{who}: shape variation (humanoid_shapes rows differ); the floor table is per shape")
    gender = int(shapes[0, 0])
    parser = {0: "smpl_parser_n", 1: "smpl_parser_m", 2: "smpl_parser_f"}[gender]
    pml = ml if isinstance(ml, MotionLibB200) else MotionLibB200.from_reference(ml, device=task.device)
    pml._sampling_batch_prob = ml._sampling_batch_prob
    return pml, smpl_ground_table(pml._motion_aa, getattr(task, parser), shapes[0, 1:].float())


class HumanoidZTaskResetB200Mixin:
    """`_reset_envs` of HumanoidReach(Z) / HumanoidSpeed(Z) / HumanoidStrike(Z) on the device.  Usage:

        class HumanoidReachZB200(HumanoidZTaskResetB200Mixin, HumanoidReachB200Mixin, HumanoidZB200Mixin, HumanoidReachZ): pass

    For StateInit Random / Start, in the reference's order (humanoid_amp_task.py:66-76, humanoid_amp.py:347-356, humanoid.py:574-587):
    the draws with the reference's own calls in the reference's order (so `torch.manual_seed` fixes them), `pulse_reset_ztask`, the
    task's `_reset_env_tensors` and `_refresh_sim_tensors` with the `_reset_rb_*` restore, the list observation of the reset envs, then
    `pulse_ztask_reset_task`.  The clips come from the reference's own `sample_motions` call (`torch.multinomial` with replacement,
    which reads nothing back to the host), so a seeded run draws the reference's numbers.  No host synchronisation.  Default / Hybrid state init go back to the reference.  The floor table is built at the first reset and again
    whenever the MotionLib's tables are replaced."""

    def _pulse_ztask_kind(self) -> str:
        if hasattr(self, "_target_states"):
            return "strike"
        if hasattr(self, "_tar_speed"):
            return "speed"
        if hasattr(self, "_tar_pos"):
            return "reach"
        raise _lib.PulseError("HumanoidZTaskResetB200Mixin serves HumanoidReach(Z), HumanoidSpeed(Z) and HumanoidStrike(Z)")

    def _pulse_ztask_setup(self) -> "ZTaskResetB200":
        ml = self._motion_lib
        if getattr(self, "_pulse_zr", None) is not None and self._pulse_zr_src is ml.gts:
            self._pulse_zr.motion_lib._sampling_batch_prob = ml._sampling_batch_prob     # follows the reference's sampling weights
            return self._pulse_zr
        pml, floor = smpl_reset_tables(self, ml, "HumanoidZTaskResetB200Mixin")
        kind = self._pulse_ztask_kind()
        kw = {}
        if kind == "strike":
            kw = dict(near_prob=self._near_prob, near_dist=self._near_dist, tar_dist_min=self._tar_dist_min, tar_dist_max=self._tar_dist_max)
        elif kind == "reach":
            kw = dict(reach_dist_max=self._tar_dist_max, tar_height_min=self._tar_height_min, tar_height_max=self._tar_height_max,
                      change_steps_min=self._tar_change_steps_min, change_steps_max=self._tar_change_steps_max)
        else:
            kw = dict(tar_speed_min=self._tar_speed_min, tar_speed_max=self._tar_speed_max, change_steps_min=self._speed_change_steps_min,
                      change_steps_max=self._speed_change_steps_max)
        self._pulse_zr = ZTaskResetB200(kind, pml, floor, upright=bool(self._has_upright_start), state_init=self._state_init.name,
                                        amp_root_height_obs=bool(self._amp_root_height_obs), dt=float(self.dt), **kw)
        self._pulse_zr_src = ml.gts
        N, dev = self.num_envs, self.device
        self._pulse_zr_draws = {"motion_ids": torch.zeros(N, dtype=torch.int64, device=dev), "phase": torch.zeros(N, device=dev),
                                "strike_u": torch.zeros(N, 4, device=dev), "task_u": torch.zeros(N, 3 if kind == "reach" else 1, device=dev),
                                "steps": torch.zeros(N, dtype=torch.int64, device=dev)}
        self._pulse_zr_obs = self._pulse_ztask_observer(kind)
        return self._pulse_zr

    def _pulse_ztask_observer(self, kind):
        """The step object whose list kernel writes the reset envs' observation rows into the task's own obs_buf (and reads its target)."""
        from .reach import ReachTaskB200
        from .ztasks import SpeedTaskB200, StrikeTaskB200
        if kind == "reach":
            o = ReachTaskB200(self.num_envs, device=self.device)
            o._tar_pos = self._tar_pos
        elif kind == "speed":
            o = SpeedTaskB200(self.num_envs, device=self.device)
            o._tar_speed = self._tar_speed
        else:
            o = StrikeTaskB200(self.num_envs, device=self.device)
        o.obs_buf = self.obs_buf
        return o

    def _reset_envs(self, env_ids):
        if self._state_init.name not in _INIT:
            return super()._reset_envs(env_ids)            # Default / Hybrid: the reference
        self._reset_default_env_ids = []
        self._reset_ref_env_ids = []
        n = len(env_ids)
        if n == 0:
            return
        r = self._pulse_ztask_setup()
        dev, kind, d = self.device, r.kind, self._pulse_zr_draws
        ids = env_ids.to(dev, torch.int64).contiguous()
        # the reference's draws, in its order: sample_motions, sample_time_interval (Random), _reset_target (strike)
        d["motion_ids"][ids] = torch.multinomial(self._motion_lib._sampling_batch_prob, num_samples=n, replacement=True).to(dev)
        if self._state_init.name == "Random":
            d["phase"][ids] = torch.rand(n, device=dev)
        if kind == "strike":
            for c in range(4):
                d["strike_u"][ids, c] = torch.rand([n], dtype=self._target_states.dtype, device=dev)
        self._state_reset_happened = True
        r.reset_envs(env_ids=ids, root_states=self._humanoid_root_states, dof_pos=self._dof_pos, dof_vel=self._dof_vel,
                     rigid_body_state=self._rigid_body_state_reshaped, progress_buf=self.progress_buf,
                     sampled_motion_ids=self._sampled_motion_ids, motion_start_times=self._motion_start_times,
                     terminate_buf=self._terminate_buf, contact_forces=self._contact_forces, amp_obs_buf=self._amp_obs_buf,
                     actor_ids=self._humanoid_actor_ids, target_states=self._target_states if kind == "strike" else None,
                     tar_actor_ids=getattr(self, "_tar_actor_ids", None), motion_ids=d["motion_ids"], phase=d["phase"],
                     strike_u=d["strike_u"] if kind == "strike" else None)
        # what _reset_ref_state_init / _set_env_state leave for the refresh and the later steps (humanoid_amp.py:478-485, :590-595)
        self._reset_ref_env_ids, self._reset_ref_motion_ids, self._reset_ref_motion_times = ids, self._sampled_motion_ids[ids], self._motion_start_times[ids]
        self._reset_rb_pos, self._reset_rb_rot = self._rigid_body_pos[ids].clone(), self._rigid_body_rot[ids].clone()
        self._reset_rb_vel, self._reset_rb_ang_vel = self._rigid_body_vel[ids].clone(), self._rigid_body_ang_vel[ids].clone()
        if kind == "speed" and hasattr(self, "power_acc"):
            self.power_acc.index_fill_(0, ids, 0.0)         # HumanoidSpeed._reset_ref_state_init (a kernel-argument scalar: no host copy)
        self._reset_env_tensors(ids)
        self._refresh_sim_tensors()
        obs_kw = {"target_states": self._target_states} if kind == "strike" else {}
        r.observe(self._pulse_zr_obs, self._rigid_body_state_reshaped, self.progress_buf, **obs_kw)
        if kind == "strike":
            return
        # _reset_task: its own draws, after the observation as in the reference
        if kind == "reach":
            d["task_u"][ids] = torch.rand([n, 3], device=dev)
            lo, hi = self._tar_change_steps_min, self._tar_change_steps_max
        else:
            d["task_u"][ids, 0] = torch.rand(n, device=dev)
            lo, hi = self._speed_change_steps_min, self._speed_change_steps_max
        d["steps"][ids] = torch.randint(low=lo, high=hi, size=(n,), device=dev, dtype=torch.int64)
        if kind == "reach":
            r.reset_task(progress_buf=self.progress_buf, change_steps=self._tar_change_steps, tar_pos=self._tar_pos, rand=d["task_u"], steps=d["steps"])
        else:
            r.reset_task(progress_buf=self.progress_buf, change_steps=self._speed_change_steps, tar_speed=self._tar_speed,
                         rand=d["task_u"].view(-1), steps=d["steps"])
