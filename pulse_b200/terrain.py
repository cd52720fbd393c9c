"""Pedestrian terrain task HumanoidPedestrianTerrain(Z) (phc/env/tasks/humanoid_pedestrian_terrain.py, `env=env_pulse_terrain`) on the
device: the height-map / trajectory observation, reward and reset of post_physics_step in one launch (`pulse_terrain_step`), waypoint
generation for reset envs (`pulse_traj_reset`, TrajGenerator.reset phc/utils/traj_generator.py:57-112) and standalone height sampling
(`pulse_terrain_heights`).  Isaac Gym keeps the physics and the terrain mesh; the heightfield is uploaded once.

  TerrainB200                          the int16 heightfield + scales (Terrain.heightsamples, :1114-1173), or a plane
  PedestrianTerrainTaskB200            explicit API with the reference's method names, mirroring SpeedTaskB200
  HumanoidPedestrianTerrainB200Mixin   overrides the reference task's methods (composes with HumanoidZB200Mixin for the Z task)

Observation = [self 358 | trajectory 2 T | heights P] (humanoid_amp_task.py:81-91, :253-268); 1402 floats for env_pulse_terrain.yaml.
"""
import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import PulseError
from .reach import SMPL_BODY_NAMES

SELF_OBS = 358
TERRAIN_OBS = SELF_OBS + 2 * 10 + 32 * 32
HEAD_BODY_ID = SMPL_BODY_NAMES.index("Head")


def _grid_points(x: np.ndarray, y: np.ndarray) -> torch.Tensor:
    """torch.meshgrid(x, y) ('ij') flattened into [len(x) * len(y), 3] fp32 offsets with z = 0 (init_*_height_points :591-688)."""
    gx, gy = np.meshgrid(x, y, indexing="ij")
    p = torch.zeros(gx.size, 3)
    p[:, 0], p[:, 1] = torch.from_numpy(gx.reshape(-1)), torch.from_numpy(gy.reshape(-1))
    return p


def square_height_points(sensor_extent: float = 2.0, sensor_res: int = 32) -> torch.Tensor:
    """init_square_height_points (:608-626)."""
    v = np.linspace(-sensor_extent, sensor_extent, sensor_res)
    return _grid_points(v, v)


def center_height_points() -> torch.Tensor:
    """init_center_height_points (:591-606): x in +-0.1, y in +-0.2, 3 x 3."""
    return _grid_points(np.linspace(-0.1, 0.1, 3), np.linspace(-0.2, 0.2, 3))


class TerrainB200:
    """The heightfield the task samples: int16 [rows, cols] (row = x cell), horizontal_scale metres per cell, vertical_scale metres per
    unit.  `heightfield=None` is a plane: every height is 0 (get_heights / get_center_heights :692-696, :721-725)."""

    def __init__(self, heightfield: Optional[torch.Tensor], horizontal_scale: float = 0.1, vertical_scale: float = 0.005, device="cuda:0"):
        self.device = torch.device(device)
        self.horizontal_scale, self.vertical_scale = float(horizontal_scale), float(vertical_scale)
        if heightfield is None:
            self.heightfield, self.rows, self.cols = None, 0, 0
            return
        hf = torch.as_tensor(heightfield)
        if hf.dim() != 2 or hf.dtype != torch.int16 or hf.shape[0] < 2 or hf.shape[1] < 2:
            raise PulseError("heightfield must be an int16 [rows >= 2, cols >= 2] array")
        self.heightfield = hf.to(self.device).contiguous()
        self.rows, self.cols = int(hf.shape[0]), int(hf.shape[1])

    @classmethod
    def from_reference(cls, terrain, device="cuda:0", terrain_type: str = "trimesh") -> "TerrainB200":
        """From the reference's `Terrain` object (heightsamples, horizontal_scale, vertical_scale); `terrain_type` 'plane' gives a plane."""
        if terrain_type == "plane":
            return cls(None, device=device)
        if terrain_type == "none":
            raise PulseError("terrainType 'none' has no heights to measure (the reference raises too, :697-698)")
        if type(terrain).__name__ == "MeshTerrain":
            raise PulseError("mesh terrain (real_mesh, MeshTerrain) is not supported")
        return cls(torch.as_tensor(terrain.heightsamples).to(torch.int16).view(-1, terrain.heightsamples.shape[-1]), terrain.horizontal_scale,
                   terrain.vertical_scale, device)

    def fill(self, a) -> None:
        a.heightfield = self.heightfield.data_ptr() if self.heightfield is not None else None
        a.hf_rows, a.hf_cols = self.rows, self.cols
        a.horizontal_scale, a.vertical_scale = self.horizontal_scale, self.vertical_scale


class PedestrianTerrainTaskB200:
    """HumanoidPedestrianTerrain (humanoid_pedestrian_terrain.py:31-896): follow a random 2-D trajectory over uneven ground, seeing a
    height map around the head.  Buffers: obs_buf [N, get_obs_size()], rew_buf, reward_raw [N, 2] (location, power), reset_buf,
    _terminate_buf, traj_verts [N, 101, 3] (TrajGenerator._verts)."""

    def __init__(self, num_envs: int, device="cuda:0", terrain: Optional[TerrainB200] = None,
                 contact_bodies: Sequence[str] = ("R_Ankle", "L_Ankle", "R_Toe", "L_Toe"), max_episode_length: int = 300, dt: float = 1.0 / 30.0,
                 num_traj_samples: int = 10, traj_sample_timestep: float = 0.5, speed_min: float = 0.0, speed_max: float = 3.0,
                 accel_max: float = 2.0, sharp_turn_prob: float = 0.02, dtheta_max: float = 2.0, height_points: Optional[torch.Tensor] = None,
                 upright: bool = True, fuzzy_target: bool = False, power_reward: bool = False, power_coefficient: float = 0.0005,
                 use_center_height: bool = True, enable_early_termination: bool = True, no_collision_check: bool = False, fail_dist: float = 4.0,
                 seed: int = 0):
        self.device, self.num_envs = torch.device(device), int(num_envs)
        dev = self.device
        self.terrain = terrain if terrain is not None else TerrainB200(None, device=dev)
        self.contact_body_mask = 0
        for n in contact_bodies:
            self.contact_body_mask |= 1 << SMPL_BODY_NAMES.index(n)
        self.max_episode_length, self.dt = int(max_episode_length), float(dt)
        self.num_traj_samples, self.traj_sample_timestep = int(num_traj_samples), float(traj_sample_timestep)
        # HumanoidTraj._build_traj_generator (humanoid_traj.py:106-114), TrajGenerator.__init__ (traj_generator.py:38-49)
        self.traj_dt = max_episode_length * dt / (_lib.TRAJ_VERTS - 1)
        self.speed_min, self.speed_max, self.accel_max, self.sharp_turn_prob, self.dtheta_max = speed_min, speed_max, accel_max, sharp_turn_prob, dtheta_max
        self.upright, self.fuzzy_target, self.power_reward, self.power_coefficient = bool(upright), bool(fuzzy_target), bool(power_reward), float(power_coefficient)
        self.use_center_height, self.enable_early_termination = bool(use_center_height), bool(enable_early_termination)
        self.no_collision_check, self.fail_dist = bool(no_collision_check), float(fail_dist)
        self.height_points = (square_height_points() if height_points is None else torch.as_tensor(height_points, dtype=torch.float32)).to(dev).contiguous()
        self.center_points = center_height_points().to(dev)
        self.seed, self._rng_offset = int(seed), 0
        self.obs_buf = torch.zeros(num_envs, self.get_obs_size(), device=dev)
        self.rew_buf = torch.zeros(num_envs, device=dev)
        self.reward_raw = torch.zeros(num_envs, 2, device=dev)
        self.reset_buf = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self._terminate_buf = torch.zeros(num_envs, dtype=torch.int64, device=dev)
        self.traj_verts = torch.zeros(num_envs, _lib.TRAJ_VERTS, 3, device=dev)
        self.lib = _lib.load()

    def get_task_obs_size(self) -> int:
        return 2 * self.num_traj_samples + int(self.height_points.shape[0])

    def get_obs_size(self) -> int:
        return SELF_OBS + self.get_task_obs_size()

    def _stream(self):
        return _lib.current_stream(self.device)

    def reset_task(self, env_ids: torch.Tensor, root_pos: torch.Tensor, rand: Optional[torch.Tensor] = None) -> None:
        """_reset_task (:480-485) -> TrajGenerator.reset(env_ids, root_pos): new waypoints starting at root_pos[i, 0:2] for env_ids[i].
        `rand` [n, 402] injects the uniform draws (layout in pulse_b200.h); otherwise Philox draws them, a fresh stream per call."""
        env_ids = env_ids.to(self.device, torch.int64).contiguous()
        n = int(env_ids.shape[0])
        if n == 0:
            return
        if root_pos.shape[0] != n or root_pos.stride(-1) != 1 or root_pos.shape[-1] < 2:
            raise PulseError("root_pos must hold one [x, y, ...] row per env id")
        if rand is not None and (tuple(rand.shape) != (n, _lib.TRAJ_DRAWS) or not rand.is_contiguous() or rand.dtype != torch.float32):
            raise PulseError(f"rand must be a contiguous fp32 [{n}, {_lib.TRAJ_DRAWS}] tensor")
        a = _lib.TrajResetArgs(env_ids=env_ids.data_ptr(), num_ids=n, init_pos=root_pos.data_ptr(), init_stride=root_pos.stride(0),
                               rand=rand.data_ptr() if rand is not None else None, seed=self.seed, offset=self._rng_offset,
                               dtheta_scale=self.dtheta_max * self.traj_dt, dspeed_scale=self.accel_max * self.traj_dt, seg_dt=self.traj_dt,
                               speed_min=self.speed_min, speed_max=self.speed_max, sharp_turn_prob=self.sharp_turn_prob, verts=self.traj_verts.data_ptr())
        self._rng_offset += _lib.TRAJ_VERTS
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_traj_reset(C.byref(a), self._stream()), "pulse_traj_reset")

    def _step_args(self, flags, rigid_body_state, root_states, progress_buf):
        if rigid_body_state.dim() != 3 or rigid_body_state.shape[1] < 24 or rigid_body_state.stride(1) != 13 or rigid_body_state.stride(2) != 1:
            raise PulseError("rigid_body_state must be a [N, B>=24, 13] view with row stride 13")
        if root_states.dim() != 2 or root_states.shape[1] < 13 or root_states.stride(1) != 1:
            raise PulseError("root_states must be a [N, 13] view with unit element stride")
        a = _lib.TerrainStepArgs(
            flags=flags, upright=int(self.upright), body_state=rigid_body_state.data_ptr(), body_env_stride=rigid_body_state.stride(0),
            root_states=root_states.data_ptr(), root_env_stride=root_states.stride(0), progress_buf=progress_buf.data_ptr(),
            max_episode_length=self.max_episode_length, contact_body_mask=self.contact_body_mask,
            enable_early_termination=int(self.enable_early_termination), no_collision_check=int(self.no_collision_check),
            fuzzy_target=int(self.fuzzy_target), power_reward=int(self.power_reward), num_traj_samples=self.num_traj_samples,
            num_height_points=int(self.height_points.shape[0]), num_center_points=int(self.center_points.shape[0]), head_body_id=HEAD_BODY_ID,
            use_center_height=int(self.use_center_height), dt=self.dt, traj_dur=_lib.TRAJ_VERTS * self.traj_dt,
            traj_sample_timestep=self.traj_sample_timestep, fail_dist=self.fail_dist, power_coefficient=self.power_coefficient,
            traj_verts=self.traj_verts.data_ptr(), height_points=self.height_points.data_ptr(), center_points=self.center_points.data_ptr(),
            obs_buf=self.obs_buf.data_ptr(), obs_stride=self.obs_buf.stride(0))
        self.terrain.fill(a)
        return a

    def _launch(self, a, n) -> None:
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_terrain_step(C.byref(a), n, self._stream()), "pulse_terrain_step")

    def post_physics_step(self, rigid_body_state: torch.Tensor, root_states: torch.Tensor, progress_buf: torch.Tensor, contact_forces: torch.Tensor,
                          dof_force: torch.Tensor, dof_vel: torch.Tensor) -> None:
        """_compute_reward (:871-896) + _compute_reset (:849-869) + _compute_observations in one launch (progress_buf already advanced).
        rigid_body_state [N, B, 13], root_states [N, 13] (the actor root state view), contact_forces [N, B, 3], dof_force [N, 69],
        dof_vel [N, 69] view."""
        a = self._step_args(_lib.STEP_ALL, rigid_body_state, root_states, progress_buf)
        a.contact_forces, a.contact_env_stride = contact_forces.data_ptr(), contact_forces.stride(0)
        a.dof_force, a.dof_force_stride = dof_force.data_ptr(), dof_force.stride(0)
        a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dof_vel.data_ptr(), dof_vel.stride(0), dof_vel.stride(1)
        a.rew_buf, a.reward_raw, a.raw_stride = self.rew_buf.data_ptr(), self.reward_raw.data_ptr(), self.reward_raw.stride(0)
        a.reset_buf, a.terminate_buf = self.reset_buf.data_ptr(), self._terminate_buf.data_ptr()
        self._launch(a, self.num_envs)

    def compute_observations(self, rigid_body_state: torch.Tensor, root_states: torch.Tensor, progress_buf: torch.Tensor,
                             env_ids: Optional[torch.Tensor] = None) -> None:
        """_compute_observations(env_ids): obs_buf rows of env_ids (all envs when None) = [self | trajectory | heights]."""
        a = self._step_args(_lib.STEP_OBS, rigid_body_state, root_states, progress_buf)
        n = self.num_envs
        if env_ids is not None:
            env_ids = env_ids.to(self.device, torch.int64).contiguous()
            n = int(env_ids.shape[0])
            if n == 0:
                return
            a.env_ids = env_ids.data_ptr()
        self._launch(a, n)

    def _heights(self, mode, root_states, points) -> torch.Tensor:
        if root_states.dim() != 2 or root_states.shape[1] < 7 or root_states.stride(1) != 1:
            raise PulseError("root_states must be [n, >=7] rows [pos 3 | quat 4] with unit element stride")
        n = int(root_states.shape[0])
        out = torch.empty(n, int(points.shape[0]), device=self.device)
        a = _lib.TerrainHeightsArgs(mode=mode, upright=int(self.upright), root_states=root_states.data_ptr(), root_stride=root_states.stride(0),
                                    num_rows=n, points=points.data_ptr(), num_points=int(points.shape[0]), heights=out.data_ptr(),
                                    heights_stride=out.stride(0))
        self.terrain.fill(a)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_terrain_heights(C.byref(a), self._stream()), "pulse_terrain_heights")
        return out

    def get_center_heights(self, root_states: torch.Tensor, env_ids=None) -> torch.Tensor:
        """get_center_heights (:690-716): [n, 9] heights around each root (pos | quat rows)."""
        return self._heights(_lib.HEIGHTS_CENTER, root_states, self.center_points)

    def get_heights(self, root_states: torch.Tensor, env_ids=None) -> torch.Tensor:
        """get_heights (:718-772): [n, P] heights of the sensor grid around each pose, rotated by its heading."""
        return self._heights(_lib.HEIGHTS_GRID, root_states, self.height_points)


def check_terrain_options(task, flags) -> None:
    """Refuses the reference options this path does not cover (a PulseError naming the option)."""
    refuse = [("divide_group", getattr(task, "_divide_group", False) or getattr(flags, "divide_group", False)),
              ("group_obs", getattr(task, "_group_obs", False)), ("velocity_map", getattr(task, "velocity_map", False)),
              ("real_mesh (MeshTerrain)", getattr(task, "real_mesh", False) or type(getattr(task, "terrain", None)).__name__ == "MeshTerrain"),
              ("has_shape_obs", getattr(task, "_has_shape_obs", False)), ("big_ankle", getattr(task, "big_ankle", False))]
    refuse += [(f"flags.{f}", getattr(flags, f, False)) for f in ("server_mode", "real_path", "fixed_path", "slow")]
    for name, on in refuse:
        if on:
            raise PulseError(f"HumanoidPedestrianTerrainB200Mixin does not support {name}")
    if not getattr(task, "_local_root_obs", True) or not getattr(task, "_root_height_obs", True):
        raise PulseError("HumanoidPedestrianTerrainB200Mixin needs local_root_obs and root_height_obs (env_pulse_terrain.yaml)")


class HumanoidPedestrianTerrainB200Mixin:
    """Mix in front of HumanoidPedestrianTerrain (or HumanoidPedestrianTerrainZ, after HumanoidZB200Mixin):

        class HumanoidPedestrianTerrainZB200(HumanoidPedestrianTerrainB200Mixin, HumanoidZB200Mixin, HumanoidPedestrianTerrainZ): pass

    The first of _compute_reward / _compute_reset / _compute_observations after a physics step runs the fused launch for all three;
    the reference's buffers (obs_buf, rew_buf, reward_raw, reset_buf, _terminate_buf, _traj_gen._verts) are shared, so every other
    method of the task keeps seeing them.  The spawn placement (_reset_ref_state_init) stays the reference's; its get_center_heights
    call runs here."""

    def _pulse_terrain(self) -> PedestrianTerrainTaskB200:
        t = getattr(self, "_pulse_terrain_obj", None)
        if t is not None:
            return t
        from .flags_compat import reference_flags
        check_terrain_options(self, reference_flags())
        if self.terrain_obs_type not in ("square", "fov", "square_fov") or not self.terrain_obs or self.terrain_obs_root != "head":
            raise PulseError("HumanoidPedestrianTerrainB200Mixin covers terrain_obs with terrain_obs_root 'head'")
        ttype = self.cfg["env"]["terrain"]["terrainType"]
        contact = [SMPL_BODY_NAMES[i] for i in self._contact_body_ids.tolist()]
        t = PedestrianTerrainTaskB200(
            self.num_envs, device=self.device, terrain=TerrainB200.from_reference(getattr(self, "terrain", None), self.device, ttype),
            contact_bodies=contact, max_episode_length=int(self.max_episode_length), dt=float(self.dt), num_traj_samples=self._num_traj_samples,
            traj_sample_timestep=self._traj_sample_timestep, speed_min=self._speed_min, speed_max=self._speed_max, accel_max=self._accel_max,
            sharp_turn_prob=self._sharp_turn_prob, height_points=self.height_points[0].float().cpu(), upright=self._has_upright_start,
            fuzzy_target=self.fuzzy_target, power_reward=self.power_reward, power_coefficient=self.power_coefficient,
            use_center_height=bool(self.cfg["env"].get("use_center_height", False)), enable_early_termination=bool(self._enable_early_termination),
            fail_dist=float(self._fail_dist))
        t.traj_verts = self._traj_gen._verts
        t.obs_buf, t.rew_buf, t.reward_raw, t.reset_buf, t._terminate_buf = self.obs_buf, self.rew_buf, self.reward_raw, self.reset_buf, self._terminate_buf
        self._pulse_terrain_obj, self._pulse_terrain_pending = t, False
        return t

    def _pulse_roots(self):
        return self._rigid_body_state_reshaped, self._humanoid_root_states

    def _pulse_fused(self):
        t = self._pulse_terrain()
        from .flags_compat import reference_flags
        t.no_collision_check = bool(getattr(reference_flags(), "no_collision_check", False))
        rb, roots = self._pulse_roots()
        t.post_physics_step(rb, roots, self.progress_buf, self._contact_forces, self.dof_force_tensor, self._dof_vel)
        self._pulse_terrain_pending = True

    def _compute_reward(self, actions):
        self._pulse_fused()

    def _compute_reset(self):
        if not getattr(self, "_pulse_terrain_pending", False):
            self._pulse_fused()

    def _compute_observations(self, env_ids=None):
        if env_ids is None and getattr(self, "_pulse_terrain_pending", False):
            self._pulse_terrain_pending = False
            return
        self._pulse_terrain_pending = False
        rb, roots = self._pulse_roots()
        self._pulse_terrain().compute_observations(rb, roots, self.progress_buf, env_ids)

    def _pulse_obs_rows(self, env_ids):
        self._compute_observations(env_ids)
        return self.obs_buf if env_ids is None else self.obs_buf[env_ids]

    def _compute_humanoid_obs(self, env_ids=None):
        return self._pulse_obs_rows(env_ids)[:, :SELF_OBS].clone()

    def _compute_task_obs(self, env_ids=None):
        return self._pulse_obs_rows(env_ids)[:, SELF_OBS:].clone()

    def _reset_task(self, env_ids):
        self._pulse_terrain().reset_task(env_ids, self._humanoid_root_states[env_ids, 0:3])

    def get_center_heights(self, root_states, env_ids=None):
        return self._pulse_terrain().get_center_heights(root_states.contiguous())

    def get_heights(self, root_states, env_ids=None):
        return self._pulse_terrain().get_heights(root_states.contiguous())
