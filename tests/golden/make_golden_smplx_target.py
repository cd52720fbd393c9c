"""Fixture for the PULSE-X reach and strike tasks (HumanoidReachZ / HumanoidStrikeZ with robot=smplx_humanoid, env_pulsex_amp.yaml):
outputs of the UNMODIFIED reference on the seeded 52-body rows of make_golden_smplx_speed.inputs plus seeded task inputs:
compute_humanoid_observations_smpl_max with upright False (humanoid.py:1675-1731), compute_location_observations /
compute_reach_reward (humanoid_reach.py:224-250) for reach bodies 17, 36 and 45, compute_humanoid_reset (humanoid.py:1573-1608),
compute_strike_observations / compute_strike_reward and the strike compute_humanoid_reset (humanoid_strike.py:270-375) for strike
bodies (35, 36, 45) under both contact sets; and of the reset methods of HumanoidReach and HumanoidStrike on a 52-body stand-in:
`_reset_ref_state_init` (root xy zeroed, humanoid_reach.py:46-48, humanoid_strike.py:147-150), `_reset_target` (strike, :124-145),
`_compute_amp_observations` / `_init_amp_obs_ref` (humanoid_amp.py:519-563, the 465-float SMPL-X rows) and `_reset_task` (reach).
The reset envs' dof and rigid-body rows are stored compact (in env id order), their AMP history for the first AMP_ENVS of them.

  * Rows 4::13: every body high, body 20 (neither a contact nor a strike body) pressing with 70 N and the target pushed with 80 N in
    x, so only the strike test of a pushed target terminates them.
  * Rows 6::13: every body high, only body 45 (a strike body above 31) pressing, the target pushed: they stand, which pins the 64-bit
    strike mask.
  * Rows 8::13: the target tipped over (rot_err < 0.2, reward 1).  Rows 10::13: the root moved away from the target (dir_speed <= 0).
  * Draws are recorded in call order (torch.multinomial / rand / randint wrapped), as make_golden_smplx_speed.py does.

  python tests/golden/make_golden_smplx_target.py     (needs the reference tree; writes tests/golden/smplx_target.npz)
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

N = 120
AMP_ENVS = 6                   # the AMP history of the first AMP_ENVS reset envs is stored (the fixture stays under 1 MB)
REACH_IDS = (17, 36, 45)
STRIKE_IDS = [35, 36, 45]
KEY_BODY_IDS = [7, 3, 36, 17]
DOF_SUBSET = [k for k in range(153) if (k // 3) not in (3, 7)]
AMP_STEPS, AMP_WIDTH = 10, 465
RESET_SEEDS = {"reach": 81, "strike": 82}


def speed_gen():
    spec = importlib.util.spec_from_file_location("make_golden_smplx_speed", os.path.join(HERE, "make_golden_smplx_speed.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def inputs(n, seed=0):
    """make_golden_smplx_speed.inputs(n, seed) with the reach target, the strike target's root state and its contact force."""
    z = speed_gen().inputs(n, seed)
    g = torch.Generator().manual_seed(seed + 1000)
    bs, cf = z["body_state"], z["contact_forces"]
    z["tar_pos"] = torch.randn(n, 3, generator=g) * torch.tensor([1.0, 1.0, 0.3]) + torch.tensor([0.0, 0.0, 1.0])
    ts = torch.zeros(n, 13)
    ts[:, 0:2] = bs[:, 0, 0:2] + torch.randn(n, 2, generator=g) * 3.0
    ts[:, 2] = 0.9 + 0.2 * torch.randn(n, generator=g)
    q = torch.randn(n, 4, generator=g)
    ts[:, 3:7] = q / q.norm(dim=-1, keepdim=True)
    ts[:, 7:13] = torch.randn(n, 6, generator=g)
    tc = torch.randn(n, 3, generator=g) * 60.0 * (torch.rand(n, 1, generator=g) < 0.5)
    for r0, body, axis in ((4, 20, 0), (6, 45, 1)):
        rows = slice(r0, None, 13)
        bs[rows, :, 2] = 1.0
        cf[rows] = 0.0
        cf[rows, body, axis] = 70.0
        tc[rows] = torch.tensor([80.0, -90.0, 0.0]) if axis == 0 else torch.tensor([10.0, -90.0, 0.0])
    ts[8::13, 3:7] = torch.tensor([0.70710678, 0.0, 0.0, 0.70710678])
    away = bs[10::13, 0, 0:2] - ts[10::13, 0:2]
    z["prev_root_pos"][10::13, 0:2] = bs[10::13, 0, 0:2] - 0.05 * away / away.norm(dim=-1, keepdim=True)
    z["target_states"], z["tar_contact_forces"] = ts, tc
    return z


def main():
    from oracle.refshim.load_reference import load_reference
    ref = load_reference()
    ref.flags.follow = False
    reach = importlib.import_module("env.tasks.humanoid_reach")
    strike = importlib.import_module("env.tasks.humanoid_strike")
    sm = speed_gen()
    z = inputs(N)
    bs, root = z["body_state"], z["body_state"][:, 0]
    empty = torch.zeros(N, 0)
    zero = torch.zeros(N, dtype=torch.long)
    out = {"num_envs": np.int64(N), "reach_ids": np.array(REACH_IDS), "strike_ids": np.array(STRIKE_IDS)}
    out["self_obs"] = ref.humanoid.compute_humanoid_observations_smpl_max(bs[..., 0:3], bs[..., 3:7], bs[..., 7:10], bs[..., 10:13], empty, empty,
                                                                          True, True, False, False, False)
    out["reach_obs"] = reach.compute_location_observations(root, z["tar_pos"])
    for b in REACH_IDS:
        out[f"reach_reward_{b}"] = reach.compute_reach_reward(bs[:, b, 0:3], root[:, 3:7], z["tar_pos"], 1.0, sm.DT)
    out["strike_obs"] = strike.compute_strike_observations(root, z["target_states"])
    out["strike_reward"] = strike.compute_strike_reward(z["target_states"][:, 0:3], z["target_states"][:, 3:7], root, z["prev_root_pos"],
                                                        torch.zeros(N, 3), sm.DT, 1.5)
    for tag, ids in (("", sm.CONTACT_IDS), ("_hi", sm.CONTACT_IDS_HI)):
        rs, tm = ref.humanoid.compute_humanoid_reset(zero, z["progress_buf"], z["contact_forces"], torch.tensor(ids), bs[..., 0:3], sm.MAX_LEN,
                                                     True, z["termination_heights"])
        out["reach_reset" + tag], out["reach_terminate" + tag] = rs, tm
        rs, tm = strike.compute_humanoid_reset(zero, z["progress_buf"], z["contact_forces"], torch.tensor(ids), bs[..., 0:3],
                                               z["tar_contact_forces"], torch.tensor(STRIKE_IDS), float(sm.MAX_LEN), True, z["termination_heights"])
        out["strike_reset" + tag], out["strike_terminate" + tag] = rs, tm
    for kind, cls in (("reach", reach.HumanoidReach), ("strike", strike.HumanoidStrike)):
        out.update(reset_fixture(kind, cls, sm))
    np.savez_compressed(os.path.join(HERE, "smplx_target.npz"), **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
    print({k: getattr(v, "shape", None) for k, v in out.items()})
    print("strike terminated:", int(out["strike_terminate"].sum()), "rows 4::13", out["strike_terminate"][4::13].tolist(),
          "rows 6::13", out["strike_terminate"][6::13].tolist())


def reset_fixture(kind, cls, sm):
    """`_reset_ref_state_init`, `_reset_target` (strike), the AMP history and `_reset_task` (reach) of a 52-body stand-in of `cls`,
    StateInit Random, has_upright_start False.  Keys <kind>_r_*."""
    from phc.utils.motion_lib_smpl import MotionLibSMPL
    from tests import smplx_speed_oracle as so
    from tests import ztask_reset_oracle as zo
    B, D, n, seed = sm.BODIES, sm.DOFS, sm.RESET_N, RESET_SEEDS[kind]
    tb = so.tables(sm.RESET_CLIPS, seed=sm.TABLE_SEED)
    betas = torch.linspace(-1.0, 1.0, 10)
    lib = MotionLibSMPL.__new__(MotionLibSMPL)
    for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs"):
        setattr(lib, k, getattr(tb, k))
    lib._motion_aa, lib._motion_lengths, lib._motion_num_frames, lib._motion_dt = tb.motion_aa, tb.lengths, tb.num_frames, tb.dt
    lib.length_starts, lib._motion_bodies, lib._motion_limb_weights = tb.length_starts, torch.zeros(sm.RESET_CLIPS, 17), torch.zeros(sm.RESET_CLIPS, 10)
    lib.num_bodies, lib._device = B, "cpu"
    lib._sampling_batch_prob = torch.tensor(sm.PROB)

    class Task(cls):
        def __init__(self):
            pass

    t = Task()
    t.device, t.humanoid_type, t.dt, t.amp_obs_v = "cpu", "smplx", zo.DT, 1
    t._state_init = next(c for c in cls.__mro__ if c.__name__ == "HumanoidAMP").StateInit.Random
    t._motion_lib, t.ref_motion_cache = lib, {}
    t.smpl_parser_n = t.smpl_parser_m = t.smpl_parser_f = so.Parser72(zo.StandInParser())
    t.humanoid_shapes = torch.cat([torch.ones(n, 1), betas.expand(n, 10)], dim=-1)
    t.humanoid_limb_and_weights = torch.zeros(n, 10)
    t._humanoid_root_states = torch.zeros(n, 13)
    t._dof_pos, t._dof_vel = torch.zeros(n, D), torch.zeros(n, D)
    rb = torch.zeros(n, B, 13)
    t._rigid_body_pos, t._rigid_body_rot, t._rigid_body_vel, t._rigid_body_ang_vel = rb[..., 0:3], rb[..., 3:7], rb[..., 7:10], rb[..., 10:13]
    t._motion_start_times, t._sampled_motion_ids = torch.zeros(n), torch.zeros(n, dtype=torch.long)
    t._body_names, t._has_upright_start = ["body%d" % i for i in range(B)], False
    t.progress_buf = torch.randint(0, 50, (n,), generator=torch.Generator().manual_seed(seed))
    t._num_amp_obs_steps, t._key_body_ids, t.dof_subset = AMP_STEPS, torch.tensor(KEY_BODY_IDS), torch.tensor(DOF_SUBSET)
    t._local_root_obs, t._amp_root_height_obs, t._has_dof_subset = True, False, True
    t._has_shape_obs_disc = t._has_limb_weight_obs_disc = False
    t._amp_obs_buf = torch.zeros(n, AMP_STEPS, AMP_WIDTH)
    t._curr_amp_obs_buf, t._hist_amp_obs_buf = t._amp_obs_buf[:, 0], t._amp_obs_buf[:, 1:]
    if kind == "strike":
        t._target_states = torch.zeros(n, 13)
        t._near_prob, t._near_dist, t._tar_dist_min, t._tar_dist_max = (zo.STRIKE[k] for k in ("near_prob", "near_dist", "tar_dist_min", "tar_dist_max"))
    else:
        t._tar_pos, t._tar_change_steps = torch.zeros(n, 3), torch.zeros(n, dtype=torch.long)
        t._tar_dist_max, t._tar_height_min, t._tar_height_max = zo.REACH["tar_dist_max"], zo.REACH["tar_height_min"], zo.REACH["tar_height_max"]
        t._tar_change_steps_min, t._tar_change_steps_max = zo.REACH["steps_min"], zo.REACH["steps_max"]
    env_ids = torch.from_numpy(np.flatnonzero(np.random.default_rng(seed).random(n) < 0.6)).long()
    rec = []
    multinomial0, rand0, randint0 = torch.multinomial, torch.rand, torch.randint

    def wrap(name, fn):
        def f(*a, **k):
            res = fn(*a, **k)
            rec.append((name, res.clone()))
            return res
        return f

    torch.manual_seed(seed)
    torch.multinomial, torch.rand, torch.randint = wrap("multinomial", multinomial0), wrap("rand", rand0), wrap("randint", randint0)
    try:
        t._reset_ref_state_init(env_ids)
        if kind == "strike":
            t._reset_target(env_ids)
        t._compute_amp_observations(env_ids)
        t._init_amp_obs_ref(env_ids, t._reset_ref_motion_ids, t._reset_ref_motion_times)
        if kind == "reach":
            t._reset_task(env_ids)
    finally:
        torch.multinomial, torch.rand, torch.randint = multinomial0, rand0, randint0
    p = kind + "_r_"
    out = {p + "env_ids": env_ids.numpy(), p + "progress": t.progress_buf.numpy(), p + "draws": np.array(" ".join(nm for nm, _ in rec)),
           p + "root_states": t._humanoid_root_states.numpy(), p + "dof_pos": t._dof_pos[env_ids].numpy(), p + "dof_vel": t._dof_vel[env_ids].numpy(),
           p + "body_state": rb[env_ids].numpy(), p + "start_times": t._motion_start_times.numpy(), p + "motion_ids": t._sampled_motion_ids.numpy(),
           p + "amp_obs": t._amp_obs_buf[env_ids[:AMP_ENVS]].numpy()}
    if kind == "strike":
        out[p + "target_states"] = t._target_states.numpy()
    else:
        out[p + "tar_pos"], out[p + "change_steps"] = t._tar_pos.numpy(), t._tar_change_steps.numpy()
    for i, (_, v) in enumerate(rec):
        out[p + f"draw{i}"] = v.numpy()
    return out


if __name__ == "__main__":
    main()
