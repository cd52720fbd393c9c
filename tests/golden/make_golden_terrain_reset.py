"""Fixture for the pedestrian terrain task's reference-state reset: the UNMODIFIED reference's `_reset_ref_state_init`
(humanoid_pedestrian_terrain.py:527-589, with `_sample_ref_state` :488-525 and the SMPL ground fix `_get_fixed_smpl_state_from_motionlib`,
humanoid_amp.py:382-430), `Terrain.sample_valid_locations` (:1175-1189) under a seeded `np.random`, `get_center_heights` (:690-716) with
`Terrain.sample_height_points` (:1200-1267), `_set_env_state` and `_compute_amp_observations` / `_init_amp_obs_ref`
(humanoid_amp.py:519-563), run on stand-ins of HumanoidPedestrianTerrain, upright and not, with StateInit Random and Start.

  * The stand-in subclasses the reference task without running its constructor and carries the tensors these methods touch.  The
    MotionLib is an un-initialised reference `MotionLibSMPL` holding the tables of `tests.ztask_reset_oracle.fixture_tables`.
  * The terrain is an un-initialised reference `Terrain` with the synthetic heightfield of make_golden_terrain.py (steps, a slope,
    noise, spikes) and the walkable table `tests.terrain_reset_oracle.walkable_table` restates from Terrain.__init__ (:1160-1171),
    which cannot run here (it builds the whole trimesh).
  * `torch.multinomial`, `torch.rand` and `np.random.randint` are wrapped to record their results in call order.  Only outputs and
    draws are stored.

  python tests/golden/make_golden_terrain_reset.py     (needs the reference tree; writes tests/golden/terrain_reset.npz)
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

N = 48
BORDER = 5                        # cells of the walkable table's border (border_size / horizontal_scale; 500 in env_pulse_terrain)
PROB = [0.3, 0.0, 0.2, 0.1, 0.0, 0.25, 0.15]
# name: (upright, state init, seed)
CASES = {"upright": (True, "Random", 51), "tilted": (False, "Random", 52), "start": (True, "Start", 53)}
BODY_NAMES = ['Pelvis', 'L_Hip', 'L_Knee', 'L_Ankle', 'L_Toe', 'R_Hip', 'R_Knee', 'R_Ankle', 'R_Toe', 'Torso', 'Spine', 'Chest', 'Neck',
              'Head', 'L_Thorax', 'L_Shoulder', 'L_Elbow', 'L_Wrist', 'L_Hand', 'R_Thorax', 'R_Shoulder', 'R_Elbow', 'R_Wrist', 'R_Hand']


def env_ids(seed):
    """About 60 % of the envs, always with env 0 and env N - 1."""
    g = np.random.default_rng(seed)
    m = g.random(N) < 0.6
    m[0] = m[-1] = True
    return torch.from_numpy(np.flatnonzero(m)).long()


def main():
    import make_golden_terrain as mgt
    from oracle import pulse_oracle as po
    from tests import terrain_reset_oracle as tro
    from tests import ztask_reset_oracle as zo
    ref, mod, _, _ = mgt._reference()
    ref.flags.follow, ref.flags.fixed, ref.flags.server_mode = False, False, False
    amp = importlib.import_module("env.tasks.humanoid_amp")
    from phc.utils.motion_lib_smpl import MotionLibSMPL

    tb, betas = zo.fixture_tables()
    hf = torch.from_numpy(mgt.heightfield())
    cx, cy = tro.walkable_table(tro.walkable_field(*hf.shape), mgt.HSCALE, BORDER)
    rec = []
    multinomial0, rand0, randint0 = torch.multinomial, torch.rand, np.random.randint

    def wrap(name, fn):
        def f(*a, **k):
            out = fn(*a, **k)
            rec.append((name, torch.as_tensor(out).clone()))
            return out
        return f

    out = {}
    for case, (upright, init, seed) in CASES.items():
        lib = MotionLibSMPL.__new__(MotionLibSMPL)
        for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs"):
            setattr(lib, k, getattr(tb, k))
        lib._motion_aa, lib._motion_lengths, lib._motion_num_frames, lib._motion_dt = tb.motion_aa, tb.lengths, tb.num_frames, tb.dt
        lib.length_starts, lib._motion_bodies, lib._motion_limb_weights = tb.length_starts, tb.motion_bodies, tb.motion_limb_weights
        lib.num_bodies, lib._device = 24, "cpu"
        lib._sampling_batch_prob = torch.tensor(PROB)

        terrain = mod.Terrain.__new__(mod.Terrain)
        terrain.type, terrain.device, terrain.heightsamples = "trimesh", "cpu", hf
        terrain.horizontal_scale, terrain.vertical_scale = mgt.HSCALE, mgt.VSCALE
        terrain.coord_x_scale, terrain.coord_y_scale, terrain.num_samples = cx, cy, int(cx.shape[0])

        class Task(mod.HumanoidPedestrianTerrain):
            def __init__(self):
                pass

        t = Task()
        t.num_envs, t.device, t.humanoid_type, t.dt = N, "cpu", "smpl", zo.DT
        t._state_init = getattr(amp.HumanoidAMP.StateInit, init)
        t._motion_lib, t.ref_motion_cache = lib, {}
        t.smpl_parser_n = t.smpl_parser_m = t.smpl_parser_f = zo.StandInParser()
        t.humanoid_shapes = torch.cat([torch.ones(N, 1), betas.expand(N, 10)], dim=-1)          # gender 1, one shape
        t.humanoid_limb_and_weights = torch.zeros(N, 10)
        t.cfg = {"env": {"terrain": {"terrainType": "trimesh"}}}
        t.terrain, t.big_ankle = terrain, False
        t.center_height_points = t.init_center_height_points()
        t._humanoid_root_states = torch.zeros(N, 13)
        t._dof_pos, t._dof_vel = torch.zeros(N, 69), torch.zeros(N, 69)
        rb = torch.zeros(N, 24, 13)
        t._rigid_body_pos, t._rigid_body_rot, t._rigid_body_vel, t._rigid_body_ang_vel = rb[..., 0:3], rb[..., 3:7], rb[..., 7:10], rb[..., 10:13]
        t._motion_start_times, t._sampled_motion_ids = torch.zeros(N), torch.zeros(N, dtype=torch.long)
        t._body_names, t._has_upright_start = BODY_NAMES, upright
        t._num_amp_obs_steps, t._key_body_ids, t.dof_subset = 10, torch.tensor(po.KEY_BODY_IDS), po.amp_dof_subset()
        t._local_root_obs, t._amp_root_height_obs, t._has_dof_subset = True, True, True
        t._has_shape_obs_disc = t._has_limb_weight_obs_disc = False
        t.amp_obs_v = 1
        t._amp_obs_buf = torch.zeros(N, 10, 196)
        t._curr_amp_obs_buf, t._hist_amp_obs_buf = t._amp_obs_buf[:, 0], t._amp_obs_buf[:, 1:]
        ids = env_ids(seed)
        torch.manual_seed(seed)
        np.random.seed(seed)
        rec.clear()
        seen = []
        sample0 = mod.Terrain.sample_height_points

        def sample(self, points, **kw):
            seen.append(points.clone())
            return sample0(self, points, **kw)
        torch.multinomial, torch.rand, np.random.randint = wrap("multinomial", multinomial0), wrap("rand", rand0), wrap("randint", randint0)
        mod.Terrain.sample_height_points = sample
        try:
            t._reset_ref_state_init(ids)
            t._compute_amp_observations(ids)
            t._init_amp_obs_ref(ids, t._reset_ref_motion_ids, t._reset_ref_motion_times)
        finally:
            torch.multinomial, torch.rand, np.random.randint = multinomial0, rand0, randint0
            mod.Terrain.sample_height_points = sample0
        p = case + "_"
        out[p + "env_ids"] = ids.numpy()
        out[p + "draws"] = np.array(" ".join(name for name, _ in rec))
        for i, (name, v) in enumerate(rec):
            out[p + f"draw{i}"] = v.numpy()
        out[p + "center_points_world"] = seen[0].numpy()
        out[p + "root_states"], out[p + "dof_pos"], out[p + "dof_vel"] = t._humanoid_root_states.numpy(), t._dof_pos.numpy(), t._dof_vel.numpy()
        out[p + "body_state"], out[p + "amp_obs"] = rb.numpy(), t._amp_obs_buf.numpy()
        # the terrain task's _reset_ref_state_init leaves _sampled_motion_ids / _motion_start_times as they were (it does not
        # write them, unlike HumanoidAMP's :484-485); the clips and start times are kept for _init_amp_obs in _reset_ref_motion_*
        out[p + "start_times"], out[p + "motion_ids"] = t._motion_start_times.numpy(), t._sampled_motion_ids.numpy()
        out[p + "ref_motion_ids"], out[p + "ref_motion_times"] = t._reset_ref_motion_ids.numpy(), t._reset_ref_motion_times.numpy()
    out["prob"] = np.array(PROB, dtype=np.float32)
    out["coord_x"], out["coord_y"] = cx.numpy(), cy.numpy()
    np.savez_compressed(os.path.join(HERE, "terrain_reset.npz"), **out)
    print("wrote terrain_reset.npz:", {c: str(out[c + "_draws"]) for c in CASES}, "locations", int(cx.shape[0]))


if __name__ == "__main__":
    main()
