"""Stand-in base class for HumanoidPedestrianTerrainB200Mixin (TEST INFRASTRUCTURE).

Carries the attributes of HumanoidPedestrianTerrain (phc/env/tasks/humanoid_pedestrian_terrain.py:31-87, humanoid_traj.py:21-39,
humanoid.py buffers) the mixin reads, with Isaac-Gym-shaped views: 26 rigid bodies and 2 actors per env."""
import types

import torch


class Terrain:
    def __init__(self, heightsamples, horizontal_scale=0.1, vertical_scale=0.005):
        self.heightsamples, self.horizontal_scale, self.vertical_scale = heightsamples, horizontal_scale, vertical_scale


class HumanoidPedestrianTerrainStandIn:
    def __init__(self, z, device, heightfield, upright=True, fuzzy=False, power=False, use_center_height=True, **options):
        from oracle import terrain_oracle as to
        n = z["body_state"].shape[0]
        self.num_envs, self.device = n, device
        self.cfg = {"env": {"terrain": {"terrainType": "trimesh"}, "use_center_height": use_center_height}}
        self.terrain = Terrain(heightfield)
        self.terrain_obs, self.terrain_obs_type, self.terrain_obs_root = True, "square", "head"
        self.height_points = to.square_height_points().expand(n, -1, -1)
        self._has_upright_start, self.fuzzy_target, self.power_reward, self.power_coefficient = upright, fuzzy, power, 0.0005
        self._divide_group, self._group_obs, self.velocity_map, self.real_mesh, self._has_shape_obs, self.big_ankle = (False,) * 6
        self._local_root_obs, self._root_height_obs = True, True
        for k, v in options.items():
            setattr(self, k, v)
        self._contact_body_ids = torch.tensor([7, 3, 8, 4], device=device)
        self.max_episode_length, self.dt, self._enable_early_termination, self._fail_dist = 300, 2 * (1.0 / 60.0), True, 4.0
        self._num_traj_samples, self._traj_sample_timestep = 10, 0.5
        self._speed_min, self._speed_max, self._accel_max, self._sharp_turn_prob = 0.0, 3.0, 2.0, 0.02
        self._traj_gen = types.SimpleNamespace(_verts=z["traj_verts"].to(device).clone())
        rb = torch.full((n, 26, 13), 5.0, device=device)
        rb[:, :24] = z["body_state"].to(device)
        self._rigid_body_state_reshaped = rb
        roots = torch.zeros(n, 2, 13, device=device)
        roots[:, 0] = z["root_states"].to(device)
        self._humanoid_root_states = roots[:, 0]
        cf = torch.zeros(n, 26, 3, device=device)
        cf[:, :24] = z["contact_forces"].to(device)
        self._contact_forces = cf
        dof_state = torch.zeros(n, 69, 2, device=device)
        dof_state[:, :, 1] = z["dof_vel"].to(device)
        self._dof_vel, self.dof_force_tensor = dof_state[:, :, 1], z["dof_force"].to(device)
        self.progress_buf = z["progress_buf"].to(device)
        self.obs_buf = torch.zeros(n, 1402, device=device)
        self.rew_buf, self.reward_raw = torch.zeros(n, device=device), torch.zeros(n, 2, device=device)
        self.reset_buf, self._terminate_buf = torch.zeros(n, dtype=torch.long, device=device), torch.zeros(n, dtype=torch.long, device=device)

    def _compute_reward(self, actions):
        raise AssertionError("the mixin must not fall through to the reference's reward")

    def _compute_reset(self):
        raise AssertionError("the mixin must not fall through to the reference's reset")

    def _compute_observations(self, env_ids=None):
        raise AssertionError("the mixin must not fall through to the reference's observations")
