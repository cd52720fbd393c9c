"""Fixture for the latent-space tasks' reference-state reset: the UNMODIFIED reference's `_reset_ref_state_init` (with
`_sample_ref_state` and the SMPL ground fix `_get_fixed_smpl_state_from_motionlib`, humanoid_amp.py:382-488), `_reset_target`
(humanoid_strike.py:124-145), `_compute_amp_observations` / `_init_amp_obs_ref` (humanoid_amp.py:519-563, :632-667) and `_reset_task`
(humanoid_reach.py:134-146, humanoid_speed.py:166-175), run on stand-ins of HumanoidReach, HumanoidSpeed (upright and not) and
HumanoidStrike with StateInit Random and Start.

  * Each stand-in subclasses the reference task without running its constructor (no simulator) and carries the tensors these methods
    touch.  The MotionLib is an un-initialised reference `MotionLibSMPL` holding the tables of `tests.ztask_reset_oracle.fixture_tables`
    (rebuilt from seeds), with zero-weight clips in its sampling probabilities.
  * SMPL model files are not part of the project: `StandInParser` (tests/ztask_reset_oracle.py) serves `get_joints_verts` for the three
    genders.  It pins how the ground fix is derived, not real SMPL geometry.
  * `torch.multinomial`, `torch.rand` and `torch.randint` are wrapped to record their results in call order, so the oracle can replay
    them as injected draws.  Only outputs and draws are stored.

  python tests/golden/make_golden_ztask_reset.py     (needs the reference tree; writes tests/golden/ztask_reset.npz)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

N = 40
PROB = [0.3, 0.0, 0.2, 0.1, 0.0, 0.25, 0.15]
# name: (task, upright, state init, seed)
CASES = {"reach": ("reach", True, "Random", 41), "reach_start": ("reach", True, "Start", 42), "speed": ("speed", True, "Random", 43),
         "speed_tilted": ("speed", False, "Random", 44), "speed_start": ("speed", True, "Start", 45), "strike": ("strike", True, "Random", 46),
         "strike_start": ("strike", True, "Start", 47)}
BODY_NAMES = ['Pelvis', 'L_Hip', 'L_Knee', 'L_Ankle', 'L_Toe', 'R_Hip', 'R_Knee', 'R_Ankle', 'R_Toe', 'Torso', 'Spine', 'Chest', 'Neck',
              'Head', 'L_Thorax', 'L_Shoulder', 'L_Elbow', 'L_Wrist', 'L_Hand', 'R_Thorax', 'R_Shoulder', 'R_Elbow', 'R_Wrist', 'R_Hand']


def main():
    from oracle.refshim.load_reference import load_reference
    ref = load_reference()
    ref.flags.follow = False               # set by run_hydra.py's flag parser in a real run
    import importlib
    from oracle import pulse_oracle as po
    from tests import ztask_reset_oracle as zo
    amp = importlib.import_module("phc.env.tasks.humanoid_amp")
    mods = {"reach": importlib.import_module("phc.env.tasks.humanoid_reach").HumanoidReach,
            "speed": importlib.import_module("phc.env.tasks.humanoid_speed").HumanoidSpeed,
            "strike": importlib.import_module("phc.env.tasks.humanoid_strike").HumanoidStrike}
    from phc.utils.motion_lib_smpl import MotionLibSMPL
    speed_mod = importlib.import_module("phc.env.tasks.humanoid_speed")
    if not hasattr(speed_mod, "quat_apply"):   # isaacgym.torch_utils.quat_apply, which the Isaac Gym stand-in does not define
        from oracle.terrain_oracle import quat_apply
        speed_mod.quat_apply = quat_apply

    tb, betas = zo.fixture_tables()
    rec = []
    multinomial0, rand0, randint0 = torch.multinomial, torch.rand, torch.randint

    def wrap(name, fn):
        def f(*a, **k):
            out = fn(*a, **k)
            rec.append((name, out.clone()))
            return out
        return f

    out = {}
    for case, (kind, upright, init, seed) in CASES.items():
        lib = MotionLibSMPL.__new__(MotionLibSMPL)
        for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs"):
            setattr(lib, k, getattr(tb, k))
        lib._motion_aa, lib._motion_lengths, lib._motion_num_frames, lib._motion_dt = tb.motion_aa, tb.lengths, tb.num_frames, tb.dt
        lib.length_starts, lib._motion_bodies, lib._motion_limb_weights = tb.length_starts, tb.motion_bodies, tb.motion_limb_weights
        lib.num_bodies, lib._device = 24, "cpu"
        lib._sampling_batch_prob = torch.tensor(PROB)

        class Task(mods[kind]):
            def __init__(self):
                pass

        t = Task()
        t.device, t.humanoid_type, t.dt = "cpu", "smpl", zo.DT
        t._state_init = getattr(amp.HumanoidAMP.StateInit, init)
        t._motion_lib, t.ref_motion_cache = lib, {}
        t.smpl_parser_n = t.smpl_parser_m = t.smpl_parser_f = zo.StandInParser()
        t.humanoid_shapes = torch.cat([torch.ones(N, 1), betas.expand(N, 10)], dim=-1)          # gender 1, one shape
        t.humanoid_limb_and_weights = torch.zeros(N, 10)
        t._humanoid_root_states = torch.zeros(N, 13)
        t._dof_pos, t._dof_vel = torch.zeros(N, 69), torch.zeros(N, 69)
        rb = torch.zeros(N, 24, 13)
        t._rigid_body_pos, t._rigid_body_rot, t._rigid_body_vel, t._rigid_body_ang_vel = rb[..., 0:3], rb[..., 3:7], rb[..., 7:10], rb[..., 10:13]
        t._motion_start_times, t._sampled_motion_ids = torch.zeros(N), torch.zeros(N, dtype=torch.long)
        t._body_names, t._has_upright_start, t.power_acc = BODY_NAMES, upright, torch.zeros(N, 2)
        t.progress_buf = torch.randint(0, 50, (N,), generator=torch.Generator().manual_seed(seed))
        t._num_amp_obs_steps, t._key_body_ids, t.dof_subset = 10, torch.tensor(po.KEY_BODY_IDS), po.amp_dof_subset()
        t._local_root_obs, t._amp_root_height_obs, t._has_dof_subset = True, False, True
        t._has_shape_obs_disc = t._has_limb_weight_obs_disc = False
        t.amp_obs_v = 1
        t._amp_obs_buf = torch.zeros(N, 10, 195)
        t._curr_amp_obs_buf, t._hist_amp_obs_buf = t._amp_obs_buf[:, 0], t._amp_obs_buf[:, 1:]
        if kind == "strike":
            t._target_states = torch.zeros(N, 13)
            t._near_prob, t._near_dist, t._tar_dist_min, t._tar_dist_max = (zo.STRIKE[k] for k in ("near_prob", "near_dist", "tar_dist_min", "tar_dist_max"))
        elif kind == "reach":
            t._tar_pos, t._tar_change_steps = torch.zeros(N, 3), torch.zeros(N, dtype=torch.long)
            t._tar_dist_max, t._tar_height_min, t._tar_height_max = zo.REACH["tar_dist_max"], zo.REACH["tar_height_min"], zo.REACH["tar_height_max"]
            t._tar_change_steps_min, t._tar_change_steps_max = zo.REACH["steps_min"], zo.REACH["steps_max"]
        else:
            t._tar_speed, t._speed_change_steps = torch.ones(N), torch.zeros(N, dtype=torch.long)
            t._tar_speed_min, t._tar_speed_max = zo.SPEED["tar_speed_min"], zo.SPEED["tar_speed_max"]
            t._speed_change_steps_min, t._speed_change_steps_max = zo.SPEED["steps_min"], zo.SPEED["steps_max"]
        g = np.random.default_rng(seed)
        env_ids = torch.from_numpy(np.flatnonzero(g.random(N) < 0.6)).long()
        torch.manual_seed(seed)
        rec.clear()
        torch.multinomial, torch.rand, torch.randint = wrap("multinomial", multinomial0), wrap("rand", rand0), wrap("randint", randint0)
        try:
            t._reset_ref_state_init(env_ids)
            if kind == "strike":
                t._reset_target(env_ids)
            t._compute_amp_observations(env_ids)
            t._init_amp_obs_ref(env_ids, t._reset_ref_motion_ids, t._reset_ref_motion_times)
            if kind != "strike":
                t._reset_task(env_ids)
        finally:
            torch.multinomial, torch.rand, torch.randint = multinomial0, rand0, randint0
        p = case + "_"
        out[p + "env_ids"], out[p + "progress"] = env_ids.numpy(), t.progress_buf.numpy()
        out[p + "draws"] = np.array(" ".join(name for name, _ in rec))
        for i, (name, v) in enumerate(rec):
            out[p + f"draw{i}"] = v.numpy()
        out[p + "root_states"], out[p + "dof_pos"], out[p + "dof_vel"] = t._humanoid_root_states.numpy(), t._dof_pos.numpy(), t._dof_vel.numpy()
        out[p + "body_state"], out[p + "amp_obs"] = rb.numpy(), t._amp_obs_buf.numpy()
        out[p + "start_times"], out[p + "motion_ids"] = t._motion_start_times.numpy(), t._sampled_motion_ids.numpy()
        if kind == "strike":
            out[p + "target_states"] = t._target_states.numpy()
        elif kind == "reach":
            out[p + "tar_pos"], out[p + "change_steps"] = t._tar_pos.numpy(), t._tar_change_steps.numpy()
        else:
            out[p + "tar_speed"], out[p + "change_steps"] = t._tar_speed.numpy(), t._speed_change_steps.numpy()
    out["prob"] = np.array(PROB, dtype=np.float32)
    np.savez_compressed(os.path.join(HERE, "ztask_reset.npz"), **out)
    print("wrote ztask_reset.npz:", {c: str(out[c + "_draws"]) for c in CASES})


if __name__ == "__main__":
    main()
