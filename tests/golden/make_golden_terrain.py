"""Fixture for the pedestrian terrain task HumanoidPedestrianTerrain(Z): outputs of the UNMODIFIED reference
(phc/env/tasks/humanoid_pedestrian_terrain.py, phc/env/util/traj_generator.py) on seeded inputs over a synthetic heightfield.

  * TrajGenerator.reset (:57-112) with its uniform / bernoulli draws injected, and calc_pos (:148-165) on the result;
  * the task methods get_center_heights, get_heights (its cells through Terrain.world_points_to_map :1191-1197), _compute_humanoid_obs,
    _compute_task_obs, _compute_reward and _compute_reset, called unbound on a stand-in task, for two option sets (upright / fuzzy /
    power / use_center_height on and off; the second over the first NB envs).

Only the reference's outputs are stored: `inputs()` and `reset_draws()` regenerate the inputs from seeds with plain torch / numpy, so
the tests rebuild them without the reference.  Isaac Gym's terrain_utils is not available, so the heightfield is synthetic: steps,
slopes, spikes and noise from a numpy seed, with body positions beyond its edges to exercise the index clip.

  python tests/golden/make_golden_terrain.py     (needs the reference tree; writes tests/golden/terrain.npz)
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

N = 257                           # envs of the first option set
NB = 96                           # envs of the second option set (the first NB rows of the same inputs)
NR = 64                           # envs of the TrajGenerator.reset / calc_pos check
DT = 2 * (1.0 / 60.0)             # controlFrequencyInv 2 x sim dt (humanoid.py:122)
MAX_LEN = 300
CONTACT_IDS = [7, 3, 8, 4]        # R_Ankle, L_Ankle, R_Toe, L_Toe
HSCALE, VSCALE = 0.1, 0.005       # Terrain.__init__ (:1121-1122)
ROWS, COLS = 200, 300
SPEED_MIN, SPEED_MAX, ACCEL_MAX, SHARP_TURN_PROB, DTHETA_MAX = 0.0, 3.0, 2.0, 0.02, 2.0   # env_pulse_terrain.yaml, humanoid_traj.py:110
TRAJ_VERTS = 101
TRAJ_DT = MAX_LEN * DT / (TRAJ_VERTS - 1)                                                  # TrajGenerator.__init__ (traj_generator.py:41)
CASES = {"a": dict(upright=True, fuzzy=False, power=False, use_center_height=True, n=N),
         "b": dict(upright=False, fuzzy=True, power=True, use_center_height=False, n=NB)}
CALC_POS_TIMES = torch.linspace(-0.5, 11.0, 37)       # both sides of the trajectory's duration (101 * TRAJ_DT = 10.1 s)
BODY_NAMES = ["Pelvis", "L_Hip", "L_Knee", "L_Ankle", "L_Toe", "R_Hip", "R_Knee", "R_Ankle", "R_Toe", "Torso", "Spine", "Chest", "Neck", "Head",
              "L_Thorax", "L_Shoulder", "L_Elbow", "L_Wrist", "L_Hand", "R_Thorax", "R_Shoulder", "R_Elbow", "R_Wrist", "R_Hand"]


def quat_apply(a, b):
    """isaacgym.torch_utils.quat_apply [3P-memory]: t = 2 (a_xyz x b); b + a_w t + a_xyz x t.  The reference's terrain module takes it
    from `isaacgym.torch_utils` (quat_apply_yaw :1571-1576, get_heights :734-742); the shim lacks it, so it is added to that module
    before the import, compiled with TorchScript like the rest of the shim."""
    shape = b.shape
    a = a.reshape(-1, 4)
    b = b.reshape(-1, 3)
    xyz = a[:, :3]
    t = xyz.cross(b, dim=-1) * 2
    return (b + a[:, 3:] * t + xyz.cross(t, dim=-1)).view(shape)


def heightfield(seed=0):
    rng = np.random.default_rng(seed)
    hf = np.zeros((ROWS, COLS), dtype=np.int16)
    x = np.arange(ROWS)[:, None]
    y = np.arange(COLS)[None, :]
    hf += (((x // 17) + (y // 23)) % 4 * 40).astype(np.int16)                 # steps of 0.2 m
    hf[100:160, 40:200] += ((x[100:160] - 100) * 6).astype(np.int16)          # slope
    hf[20:80, 200:280] += rng.integers(-20, 20, size=(60, 80)).astype(np.int16)   # noise
    sp = rng.integers(0, [ROWS, COLS], size=(300, 2))
    hf[sp[:, 0], sp[:, 1]] = 600                                               # spikes of 3 m: exercise the +-3 m clip
    return hf


def _unit(q):
    return q / q.norm(dim=-1, keepdim=True)


def _reference():
    from oracle.refshim.load_reference import load_reference
    ref = load_reference()
    importlib.import_module("isaacgym.torch_utils").quat_apply = torch.jit.script(quat_apply)
    mod = importlib.import_module("env.tasks.humanoid_pedestrian_terrain")
    tg = importlib.import_module("env.util.traj_generator")
    traj = importlib.import_module("env.tasks.humanoid_traj")
    return ref, mod, tg, traj


class _InjectDraws:
    """Makes torch.rand / torch.bernoulli return the given draws, in the order TrajGenerator.reset asks for them (:61-73): turn angles,
    sharp-turn angles, the sharp-turn bernoulli (u < p), the heading, speed changes, the initial speed."""

    def __init__(self, draws, p):
        s = TRAJ_VERTS - 1
        self.rand = [draws[:, 0:s], draws[:, s:2 * s], draws[:, 4 * s], draws[:, 3 * s:4 * s], draws[:, 4 * s + 1]]
        self.bern = [(draws[:, 2 * s:3 * s] < p).float()]

    def __enter__(self):
        self._r, self._b = torch.rand, torch.bernoulli
        torch.rand = lambda *a, **k: self.rand.pop(0).clone()
        torch.bernoulli = lambda *a, **k: self.bern.pop(0).clone()
        return self

    def __exit__(self, *exc):
        torch.rand, torch.bernoulli = self._r, self._b
        assert exc[0] is not None or (not self.rand and not self.bern), "TrajGenerator.reset consumed a different number of draws"


def make_traj_gen(tg, num_envs):
    """TrajGenerator with the state its __init__ sets (:38-55); the constructor itself calls np.int, which numpy >= 1.24 removed."""
    g = tg.TrajGenerator.__new__(tg.TrajGenerator)
    g._device = "cpu"
    g._dt = TRAJ_DT
    g._dtheta_max, g._speed_min, g._speed_max, g._accel_max, g._sharp_turn_prob = DTHETA_MAX, SPEED_MIN, SPEED_MAX, ACCEL_MAX, SHARP_TURN_PROB
    g._verts_flat = torch.zeros((num_envs * TRAJ_VERTS, 3), dtype=torch.float32)
    g._verts = g._verts_flat.view((num_envs, TRAJ_VERTS, 3))
    return g


def reset_draws(seed=5):
    """[NR, 402] uniform draws in the layout of pulse_traj_reset and NR initial root positions; a few coins force sharp turns."""
    g = torch.Generator().manual_seed(seed)
    d = torch.rand(NR, 4 * (TRAJ_VERTS - 1) + 2, generator=g)
    d[::5, 2 * (TRAJ_VERTS - 1) + 7] = 0.0
    init = torch.rand(NR, 3, generator=g) * 40.0 - 10.0
    return d, init


def _unit_xy(v):
    return v / v.norm(dim=-1, keepdim=True)


def inputs(seed=0):
    """The step inputs for N envs, from seeds with plain torch arithmetic: trajectories are random walks (no transcendental functions,
    so they rebuild bit for bit); the rigid-body root sits near the trajectory point, every 4th env 3.9 / 4.1 m from it (either side of
    fail_dist) and every 9th 9 m away."""
    g = torch.Generator().manual_seed(seed)
    p0 = torch.rand(N, 3, generator=g) * torch.tensor([ROWS * HSCALE + 4, COLS * HSCALE + 4, 0.0]) - torch.tensor([2.0, 2.0, -0.9])
    verts = torch.zeros(N, TRAJ_VERTS, 3)
    verts[:, 0, 0:2] = p0[:, 0:2]
    verts[:, 1:, 0:2] = p0[:, None, 0:2] + torch.cumsum((torch.rand(N, TRAJ_VERTS - 1, 2, generator=g) * 2 - 1) * 0.25, dim=1)
    progress = torch.randint(0, 310, (N,), generator=g)
    progress[:6] = torch.tensor([0, 1, 2, 0, 1, 2])
    progress[6:12] = torch.tensor([303, 305, 309, 299, 298, 310])               # past the trajectory's end / at max length
    from oracle.terrain_oracle import traj_calc_pos
    tar = traj_calc_pos(verts, torch.arange(N), progress * DT, TRAJ_DT)
    direction = _unit_xy(torch.randn(N, 2, generator=g))
    dist = torch.rand(N, generator=g) * 2.0
    dist[1::4] = torch.where(torch.arange(N)[1::4] % 8 == 1, 3.9, 4.1)
    dist[::9] = 9.0
    root = torch.cat([tar[:, 0:2] + dist[:, None] * direction, 0.9 + torch.rand(N, 1, generator=g) * 0.6], dim=-1)
    bs = torch.zeros(N, 24, 13)
    bs[..., 0:3] = root[:, None] + torch.randn(N, 24, 3, generator=g) * 0.3
    bs[:, 0, 0:3] = root
    bs[:, 13, 2] += 0.5                                                      # the head above the pelvis
    bs[..., 3:7] = _unit(torch.randn(N, 24, 4, generator=g))
    bs[..., 7:13] = torch.randn(N, 24, 6, generator=g)
    actor = bs[:, 0].clone()
    actor[::7, 0:3] += torch.randn(len(actor[::7]), 3, generator=g) * 0.3       # actor root state differs from the rigid body
    actor[::7, 3:7] = _unit(torch.randn(len(actor[::7]), 4, generator=g))
    actor[3::4, 0:2] = tar[3::4, 0:2] + 0.03                                   # inside the fuzzy radius
    contact = torch.zeros(N, 24, 3)
    hit = torch.randint(0, 24, (N, 3), generator=g)
    mag = 35 + torch.rand(N, 3, generator=g) * 30                              # each either side of 50
    d = _unit(torch.randn(N, 3, 3, generator=g))
    for k in range(3):
        sel = torch.arange(N) % (k + 2) == 0
        contact[sel, hit[sel, k]] += d[sel, k] * mag[sel, k:k + 1]
    dof_force, dof_vel = torch.randn(N, 69, generator=g) * 30, torch.randn(N, 69, generator=g)
    return dict(traj_verts=verts, progress_buf=progress, body_state=bs, root_states=actor, contact_forces=contact, dof_force=dof_force,
                dof_vel=dof_vel, heightfield=torch.from_numpy(heightfield()))


def case_inputs(z, n):
    """The first n envs of the inputs (the heightfield is shared)."""
    return {k: (v if k == "heightfield" else v[:n]) for k, v in z.items()}


def stand_ins(mod, traj, tg, z, case):
    class TerrainStandIn:
        world_points_to_map = mod.Terrain.world_points_to_map

        def __init__(self):
            self.heightsamples, self.horizontal_scale, self.vertical_scale, self.seen = z["heightfield"], HSCALE, VSCALE, []

        def sample_height_points(self, points, **kw):
            self.seen.append(points.clone())
            return mod.Terrain.sample_height_points(self, points, **kw)

    cls = mod.HumanoidPedestrianTerrain

    class Task:
        pass
    for name in ("get_center_heights", "get_heights", "get_head_pose", "_compute_humanoid_obs", "_compute_task_obs", "_compute_reward",
                 "_compute_reset", "init_center_height_points", "init_square_height_points"):
        setattr(Task, name, getattr(cls, name))
    Task._fetch_traj_samples = traj.HumanoidTraj._fetch_traj_samples
    t = Task()
    n = z["body_state"].shape[0]
    t.num_envs, t.device, t.humanoid_type, t.sensor_extent, t.sensor_res = n, "cpu", "smpl", 2, 32
    t.cfg = {"env": {"terrain": {"terrainType": "trimesh"}, "use_center_height": case["use_center_height"]}}
    t.center_height_points = t.init_center_height_points()
    t.height_points = t.init_square_height_points()
    t.terrain = TerrainStandIn()
    t._has_upright_start, t.fuzzy_target, t.power_reward, t.power_coefficient = case["upright"], case["fuzzy"], case["power"], 0.0005
    t.velocity_map, t._divide_group, t._group_obs, t._disable_group_obs = False, False, False, True
    bs = z["body_state"]
    t._rigid_body_pos, t._rigid_body_rot, t._rigid_body_vel, t._rigid_body_ang_vel = bs[..., 0:3], bs[..., 3:7], bs[..., 7:10], bs[..., 10:13]
    t.humanoid_shapes, t.humanoid_limb_and_weights = torch.zeros(n, 0), torch.zeros(n, 0)
    t._root_height_obs, t._local_root_obs, t._has_shape_obs, t._has_limb_weight_obs = True, True, False, False
    t._humanoid_root_states = z["root_states"]
    t.progress_buf, t.dt, t._num_traj_samples, t._traj_sample_timestep = z["progress_buf"], DT, 10, 0.5
    t._traj_gen = make_traj_gen(tg, n)
    t._traj_gen._verts[:] = z["traj_verts"]
    t.terrain_obs, t.terrain_obs_root, t.height_meas_scale, t._body_names = True, "head", 5, BODY_NAMES
    t.dof_force_tensor, t._dof_vel = z["dof_force"], z["dof_vel"]
    t.rew_buf, t.reward_raw = torch.zeros(n), torch.zeros(n, 2)
    t.reset_buf, t._terminate_buf = torch.zeros(n, dtype=torch.long), torch.zeros(n, dtype=torch.long)
    t._contact_forces, t._contact_body_ids = z["contact_forces"], torch.tensor(CONTACT_IDS)
    t.max_episode_length, t._fail_dist, t._enable_early_termination, t._termination_heights = MAX_LEN, 4.0, True, torch.full((24,), 0.15)
    return t


def main():
    ref, mod, tg, traj = _reference()
    ref.flags.divide_group = ref.flags.real_path = False
    out = {}
    # TrajGenerator.reset with injected draws, then calc_pos on both sides of the end of the trajectory
    draws, init = reset_draws()
    gen = make_traj_gen(tg, NR)
    with _InjectDraws(draws, SHARP_TURN_PROB):
        gen.reset(torch.arange(NR), init)
    out["traj_reset_verts"] = gen._verts.numpy().copy()
    ids = torch.arange(NR).repeat_interleave(len(CALC_POS_TIMES))
    out["calc_pos"] = gen.calc_pos(ids, CALC_POS_TIMES.repeat(NR)).view(NR, len(CALC_POS_TIMES), 3).numpy()
    full = inputs()
    for name, case in CASES.items():
        z = case_inputs(full, case["n"])
        t = stand_ins(mod, traj, tg, z, case)
        t._compute_reward(None)
        t._compute_reset()
        out[f"{name}_rew"], out[f"{name}_reward_raw"] = t.rew_buf.numpy(), t.reward_raw.numpy()
        out[f"{name}_reset"], out[f"{name}_terminate"] = t.reset_buf.numpy(), t._terminate_buf.numpy()
        out[f"{name}_self_obs"] = t._compute_humanoid_obs().numpy()
        out[f"{name}_task_obs"] = t._compute_task_obs().numpy()
        out[f"{name}_center_heights"] = t.get_center_heights(torch.cat([z["body_state"][:, 0, 0:3], z["body_state"][:, 0, 3:7]], dim=-1)).numpy()
        # the spawn lift of _reset_ref_state_init samples the centers at the actor roots
        out[f"{name}_root_center_heights"] = t.get_center_heights(z["root_states"][:, 0:7]).numpy()
        if name == "a":   # the cells of the head-pose height map, int16 (ROWS, COLS < 2^15); the heights follow from them
            t.terrain.seen.clear()
            t.get_heights(t.get_head_pose())
            px, py = mod.Terrain.world_points_to_map(t.terrain, t.terrain.seen[-1])
            out["a_px"], out["a_py"] = px.view(N, -1).short().numpy(), py.view(N, -1).short().numpy()
    np.savez_compressed(os.path.join(HERE, "terrain.npz"), **out)
    print({k: v.shape for k, v in out.items()})
    for name in CASES:
        print(name, "terminated", int(out[f"{name}_terminate"].sum()), "reset", int(out[f"{name}_reset"].sum()))


if __name__ == "__main__":
    main()
