"""Reference-state reset of the pedestrian terrain task HumanoidPedestrianTerrain(Z) on the device (`pulse_reset_terrain`,
`pulse_terrain_step` over the reset list, `pulse_traj_reset_list`): `HumanoidAMPTask._reset_envs` for StateInit Random / Start and the
SMPL humanoid, without the reference's boolean-mask indexing, its host `np.random.randint` round trip, its SMPL mesh forward (the ground
fix, as in `pulse_b200.ztask_reset`) and its separate height lookup.

Call order of one reset, as in the reference (humanoid.py:574-587, humanoid_amp.py:347-356, humanoid_amp_task.py:73-76):
`reset_envs` (clip, start time, ground fix, spawn on a walkable cell lifted by the mean center height, simulator views, counters, AMP
history), the simulator's refresh, `observe` (the reset envs' observation rows, which still sample the previous episode's waypoints,
seen from the new root), then `reset_task` (new waypoints from the new root).  Draws are injected per env or made by Philox4x32-10 in
the kernels (word layout: include/pulse_b200.h).  No call reads anything back to the host.
"""
import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from .motion_lib import MotionLibB200
from .terrain import PedestrianTerrainTaskB200, TerrainB200, center_height_points
from .ztask_reset import ZTaskResetB200, smpl_reset_tables


class TerrainResetB200(ZTaskResetB200):
    """The reset of the terrain task over N envs.  `floor` is the per-frame table of `smpl_ground_table`; `terrain` the heightfield
    (a plane is refused: the reference builds no walkable table for it and cannot spawn on it); `coord_x` / `coord_y` the walkable
    table (`Terrain.coord_x_scale` / `coord_y_scale`, metres); `upright` = _has_upright_start; `amp_root_height_obs` chooses the 196-
    (env_pulse_terrain.yaml) or 195-float AMP rows."""

    def __init__(self, motion_lib: MotionLibB200, floor: torch.Tensor, terrain: TerrainB200, coord_x: torch.Tensor, coord_y: torch.Tensor, *,
                 upright: bool = True, amp_root_height_obs: bool = True, dt: float = float(torch.tensor(1.0 / 60.0, dtype=torch.float32) * 2),
                 center_points: Optional[torch.Tensor] = None):
        super().__init__("reach", motion_lib, floor, upright=upright, state_init="Random", amp_root_height_obs=amp_root_height_obs, dt=dt)
        self.kind, self.pose_mode = "terrain", _lib.ZPOSE_AS_IS     # the terrain task places the root itself; it always samples t0
        if terrain.heightfield is None:
            raise _lib.PulseError("plane terrain: the reference builds no walkable table for a plane and cannot spawn on it")
        if terrain.device != self.device:
            raise _lib.PulseError(f"the terrain lives on {terrain.device}, the MotionLib on {self.device}")
        self.terrain = terrain
        cx, cy = (torch.as_tensor(c).to(self.device, torch.float32).contiguous() for c in (coord_x, coord_y))
        if cx.dim() != 1 or cx.shape != cy.shape or cx.shape[0] < 1 or cx.shape[0] >= 2 ** 32:
            raise _lib.PulseError("coord_x / coord_y must be two equally long, non-empty [L] walkable tables")
        self.coord_x, self.coord_y, self.num_locations = cx, cy, int(cx.shape[0])
        pts = center_height_points() if center_points is None else torch.as_tensor(center_points, dtype=torch.float32)
        if pts.dim() != 2 or pts.shape[1] != 3 or not 1 <= pts.shape[0] <= 32:
            raise _lib.PulseError("center_points must be [P <= 32, 3]")
        self.center_points = pts.to(self.device).contiguous()
        self._traj_calls = 0

    @classmethod
    def from_reference(cls, terrain, motion_lib: MotionLibB200, floor: torch.Tensor, terrain_type: str = "trimesh", **kw) -> "TerrainResetB200":
        """From the reference's `Terrain` (heightsamples, scales, and the walkable table `coord_x_scale` / `coord_y_scale` that its
        constructor builds, humanoid_pedestrian_terrain.py:1160-1171).  'plane' and 'none' are refused: `Terrain.__init__` returns
        before it builds the table."""
        if terrain_type in ("plane", "none"):
            raise _lib.PulseError(f"terrainType {terrain_type!r}: the reference builds no walkable table for it and cannot spawn on it")
        t = TerrainB200.from_reference(terrain, motion_lib._device, terrain_type)
        return cls(motion_lib, floor, t, torch.as_tensor(terrain.coord_x_scale), torch.as_tensor(terrain.coord_y_scale), **kw)

    def _workspace(self, N: int) -> Dict[str, torch.Tensor]:
        ws = super()._workspace(N)
        if "loc_ids" not in ws:
            ws["loc_ids"] = torch.zeros(N, dtype=torch.int64, device=self.device)
        return ws

    def reset_envs(self, *, root_states: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, rigid_body_state: torch.Tensor,
                   progress_buf: torch.Tensor, sampled_motion_ids: torch.Tensor, motion_start_times: torch.Tensor,
                   reset_buf: Optional[torch.Tensor] = None, env_ids: Optional[torch.Tensor] = None, terminate_buf: Optional[torch.Tensor] = None,
                   contact_forces: Optional[torch.Tensor] = None, amp_obs_buf: Optional[torch.Tensor] = None,
                   actor_ids: Optional[torch.Tensor] = None, motion_ids: Optional[torch.Tensor] = None, motion_u: Optional[torch.Tensor] = None,
                   phase: Optional[torch.Tensor] = None, loc_ids: Optional[torch.Tensor] = None, seed: int = 0, offset: int = 0,
                   offset_dev: Optional[torch.Tensor] = None, amp_fresh: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """`pulse_reset_terrain` for the envs of `reset_buf` (mask) or the ascending `env_ids` (int64 list): the arguments of
        `ZTaskResetB200.reset_envs` (no target actor), plus `loc_ids` int64 [N], the injected walkable-table index per env (the
        reference's `np.random.randint(0, num_samples)`), or None: Philox word z of (seed, env, offset [+ *offset_dev]); `amp_fresh` as there.  Returns the
        workspace {'env_list', 'actor_list', 'count', 'loc_ids'} (device; loc_ids holds the location index of each reset env)."""
        N = int(progress_buf.shape[0])
        a, ws = self._args(root_states=root_states, dof_pos=dof_pos, dof_vel=dof_vel, rigid_body_state=rigid_body_state, progress_buf=progress_buf,
                           sampled_motion_ids=sampled_motion_ids, motion_start_times=motion_start_times, reset_buf=reset_buf, env_ids=env_ids,
                           terminate_buf=terminate_buf, contact_forces=contact_forces, amp_obs_buf=amp_obs_buf, actor_ids=actor_ids,
                           target_states=None, tar_actor_ids=None, motion_ids=motion_ids, motion_u=motion_u, phase=phase, strike_u=None,
                           seed=seed, offset=offset, offset_dev=offset_dev, amp_fresh=amp_fresh)
        s = _lib.TerrainSpawnArgs()
        self.terrain.fill(s)
        s.center_points, s.num_center_points = self.center_points.data_ptr(), int(self.center_points.shape[0])
        s.coord_x, s.coord_y, s.num_locations = self.coord_x.data_ptr(), self.coord_y.data_ptr(), self.num_locations
        if loc_ids is not None:
            if loc_ids.dtype != torch.int64 or not loc_ids.is_contiguous() or loc_ids.shape != (N,) or loc_ids.device != self.device:
                raise _lib.PulseError(f"loc_ids must be contiguous int64 [{N}] on {self.device}")
            s.loc_ids_in = loc_ids.data_ptr()
        s.loc_ids_out = ws["loc_ids"].data_ptr()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_reset_terrain(self.motion_lib.handle, C.byref(a), C.byref(s), N, _lib.current_stream(self.device)),
                       "pulse_reset_terrain")
        return ws

    def observe(self, task: PedestrianTerrainTaskB200, rigid_body_state: torch.Tensor, root_states: torch.Tensor,
                progress_buf: torch.Tensor) -> None:
        """_compute_observations(env_ids) of the envs of the last `reset_envs`, after the simulator's refresh: `task.obs_buf` rows of
        the listed envs, by `pulse_terrain_step` (PULSE_STEP_OBS) over the device-side list and count.  The trajectory samples come
        from `task.traj_verts` as they are, i.e. the previous episode's waypoints, as in the reference."""
        if self._ws is None:
            raise _lib.PulseError("observe follows reset_envs")
        N = int(progress_buf.shape[0])
        if task.num_envs != N:
            raise _lib.PulseError(f"the task has {task.num_envs} envs, the reset {N}")
        a = task._step_args(_lib.STEP_OBS, rigid_body_state, root_states, progress_buf)
        a.env_ids, a.env_count = self._ws["env_list"].data_ptr(), self._ws["count"].data_ptr()
        task._launch(a, N)

    def reset_task(self, task: PedestrianTerrainTaskB200, root_states: torch.Tensor, rand: Optional[torch.Tensor] = None,
                   seed: Optional[int] = None, offset: Optional[int] = None, offset_dev: Optional[torch.Tensor] = None) -> None:
        """_reset_task (:480-485) -> TrajGenerator.reset of the envs of the last `reset_envs`, from root_states[e, 0:2], into
        `task.traj_verts`, with the task's trajectory parameters.  `rand` [N, PULSE_TRAJ_DRAWS] injects the draws per ENV; otherwise
        Philox on (seed, env + 4 * 2^32, 101 * (offset [+ *offset_dev]) + k).  seed defaults to the task's, offset to a count of this
        object's calls."""
        if self._ws is None:
            raise _lib.PulseError("reset_task follows reset_envs")
        N = int(task.traj_verts.shape[0])
        if root_states.dim() != 2 or root_states.shape[0] != N or root_states.shape[1] < 2 or root_states.stride(1) != 1:
            raise _lib.PulseError(f"root_states must be an [{N}, >= 2] view with contiguous rows")
        if rand is not None and (tuple(rand.shape) != (N, _lib.TRAJ_DRAWS) or not rand.is_contiguous() or rand.dtype != torch.float32):
            raise _lib.PulseError(f"rand must be a contiguous fp32 [{N}, {_lib.TRAJ_DRAWS}] tensor")
        if offset is None:
            offset, self._traj_calls = self._traj_calls, self._traj_calls + 1
        a = _lib.TrajListArgs(env_list=self._ws["env_list"].data_ptr(), count=self._ws["count"].data_ptr(), root_states=root_states.data_ptr(),
                              root_env_stride=root_states.stride(0), rand=rand.data_ptr() if rand is not None else None,
                              seed=int(task.seed if seed is None else seed) & (2 ** 64 - 1), offset=int(offset) & (2 ** 64 - 1),
                              offset_dev=offset_dev.data_ptr() if offset_dev is not None else None,
                              dtheta_scale=task.dtheta_max * task.traj_dt, dspeed_scale=task.accel_max * task.traj_dt, seg_dt=task.traj_dt,
                              speed_min=task.speed_min, speed_max=task.speed_max, sharp_turn_prob=task.sharp_turn_prob,
                              verts=task.traj_verts.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_traj_reset_list(C.byref(a), N, _lib.current_stream(self.device)), "pulse_traj_reset_list")


class HumanoidPedestrianTerrainResetB200Mixin:
    """`_reset_envs` of HumanoidPedestrianTerrain(Z) on the device.  Usage:

        class HumanoidPedestrianTerrainZB200(HumanoidPedestrianTerrainResetB200Mixin, HumanoidPedestrianTerrainB200Mixin, HumanoidZB200Mixin,
                                             HumanoidPedestrianTerrainZ): pass

    For StateInit Random / Start (the terrain task samples the start time for both), in the reference's order: the reference's own
    draws in its order (`torch.multinomial` clips, `torch.rand` phases, the host `np.random.randint` location indices, uploaded from
    pinned memory without a read-back), `pulse_reset_terrain`, the `_reset_*` bookkeeping, `_reset_env_tensors`, `_refresh_sim_tensors`
    with the `_reset_rb_*` restore, the list observation, then the waypoints (Philox, as HumanoidPedestrianTerrainB200Mixin's
    `_reset_task`).  Default / Hybrid state init go back to the reference."""

    def _pulse_terrain_reset_setup(self) -> TerrainResetB200:
        ml = self._motion_lib
        if getattr(self, "_pulse_tr", None) is not None and self._pulse_tr_src is ml.gts:
            self._pulse_tr.motion_lib._sampling_batch_prob = ml._sampling_batch_prob
            return self._pulse_tr
        from .flags_compat import reference_flags
        who = "HumanoidPedestrianTerrainResetB200Mixin"
        flags = reference_flags()
        for name, on in (("flags.fixed", getattr(flags, "fixed", False)), ("flags.server_mode", getattr(flags, "server_mode", False)),
                         ("big_ankle", getattr(self, "big_ankle", False)),
                         ("mesh terrain (real_mesh, MeshTerrain)", getattr(self, "real_mesh", False) or type(getattr(self, "terrain", None)).__name__ == "MeshTerrain")):
            if on:
                raise _lib.PulseError(f"{who} does not support {name}")
        pml, floor = smpl_reset_tables(self, ml, who)
        self._pulse_tr = TerrainResetB200.from_reference(self.terrain, pml, floor, self.cfg["env"]["terrain"]["terrainType"],
                                                         upright=bool(self._has_upright_start), amp_root_height_obs=bool(self._amp_root_height_obs),
                                                         dt=float(self.dt))
        self._pulse_tr_src = ml.gts
        N, dev = self.num_envs, self.device
        self._pulse_tr_draws = {"motion_ids": torch.zeros(N, dtype=torch.int64, device=dev), "phase": torch.zeros(N, device=dev),
                                "loc_ids": torch.zeros(N, dtype=torch.int64, device=dev), "clip": torch.zeros(N, dtype=torch.int64, device=dev),
                                "t0": torch.zeros(N, device=dev)}
        return self._pulse_tr

    def _reset_envs(self, env_ids):
        if self._state_init.name not in ("Random", "Start"):
            return super()._reset_envs(env_ids)            # Default / Hybrid: the reference
        self._reset_default_env_ids = []
        self._reset_ref_env_ids = []
        n = len(env_ids)
        if n == 0:
            return
        r = self._pulse_terrain_reset_setup()
        dev, d = self.device, self._pulse_tr_draws
        ids = env_ids.to(dev, torch.int64).contiguous()
        # the reference's draws, in its order: sample_motions, sample_time_interval, sample_valid_locations
        d["motion_ids"][ids] = torch.multinomial(self._motion_lib._sampling_batch_prob, num_samples=n, replacement=True).to(dev)
        d["phase"][ids] = torch.rand(n, device=dev)
        loc = torch.from_numpy(np.random.randint(0, r.num_locations, size=n).astype(np.int64)).pin_memory()
        d["loc_ids"][ids] = loc.to(dev, non_blocking=True)
        self._state_reset_happened = True
        r.reset_envs(env_ids=ids, root_states=self._humanoid_root_states, dof_pos=self._dof_pos, dof_vel=self._dof_vel,
                     rigid_body_state=self._rigid_body_state_reshaped, progress_buf=self.progress_buf,
                     sampled_motion_ids=d["clip"], motion_start_times=d["t0"], terminate_buf=self._terminate_buf,
                     contact_forces=self._contact_forces, amp_obs_buf=self._amp_obs_buf, actor_ids=self._humanoid_actor_ids,
                     motion_ids=d["motion_ids"], phase=d["phase"], loc_ids=d["loc_ids"])
        # what _reset_ref_state_init / _set_env_state leave for the refresh and the later steps (:583-585, humanoid_amp.py:590-595).
        # Unlike HumanoidAMP's, the terrain task's _reset_ref_state_init does not write _sampled_motion_ids / _motion_start_times,
        # so the kernel writes the clips and start times into the mixin's own buffers.
        self._reset_ref_env_ids, self._reset_ref_motion_ids, self._reset_ref_motion_times = ids, d["clip"][ids], d["t0"][ids]
        self._reset_rb_pos, self._reset_rb_rot = self._rigid_body_pos[ids].clone(), self._rigid_body_rot[ids].clone()
        self._reset_rb_vel, self._reset_rb_ang_vel = self._rigid_body_vel[ids].clone(), self._rigid_body_ang_vel[ids].clone()
        self._reset_env_tensors(ids)
        self._refresh_sim_tensors()
        t = self._pulse_terrain()
        r.observe(t, self._rigid_body_state_reshaped, self._humanoid_root_states, self.progress_buf)
        self._pulse_terrain_pending = False
        r.reset_task(t, self._humanoid_root_states)
