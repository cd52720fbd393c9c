"""Fixture for the PULSE-X speed task (HumanoidSpeedZ with robot=smplx_humanoid, env_pulsex_amp.yaml): outputs of the UNMODIFIED
reference's compute_humanoid_observations_smpl_max with upright False (humanoid.py:1675-1731, has_upright_start False),
remove_base_rot (:1617-1620), compute_speed_observations / compute_speed_reward (humanoid_speed.py:310-343) and compute_humanoid_reset
(humanoid.py:1573-1608) on seeded synthetic states of the 52-body SMPL-X humanoid, and of its reset methods: HumanoidSpeed's
`_reset_ref_state_init` (`_sample_ref_state` with the face-x adjustment and the SMPL ground fix, humanoid_speed.py:247-270,
humanoid_amp.py:382-488) and `_reset_task` (:166-175) on a synthetic 52-body MotionLib.

  * Only body indices enter: the contact bodies are given as indices into the SMPLH_MUJOCO_NAMES order (R_Ankle, L_Ankle, R_Toe, L_Toe
    under CONTACT_IDS below), so neither this generator nor the tests need smpl_sim's name list; the reset stand-in's `_body_names`
    are placeholders (only their count is read).  CONTACT_IDS_HI adds bodies above 31, and rows 2::17 have body 40 alone low and
    pressed, so they fall under CONTACT_IDS and stand under CONTACT_IDS_HI: the 64-bit contact mask is pinned.
  * The reset stand-in subclasses HumanoidSpeed without its constructor (no simulator) and holds an un-initialised reference
    MotionLibSMPL with the tables of `tests.smplx_speed_oracle.tables`; the SMPL parser is the seeded stand-in of
    tests/ztask_reset_oracle.py fed the first 72 pose columns (`Parser72`).  torch.multinomial / rand / randint are wrapped to record
    their results in call order, so the tests replay them as injected draws.
  * Root rotations are drawn far from upright (random unit quaternions), so the self observation's heading (of remove_base_rot(root))
    and the task observation's heading (of the raw root) differ in every row.

  python tests/golden/make_golden_smplx_speed.py     (needs the reference tree; writes tests/golden/smplx_speed.npz)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

BODIES, DOFS = 52, 153
CONTACT_IDS = [7, 3, 8, 4]        # R_Ankle, L_Ankle, R_Toe, L_Toe: the SMPL-H / SMPL-X MuJoCo order starts with SMPL's first 22 bodies
CONTACT_IDS_HI = [7, 3, 8, 4, 33, 40, 51]
RESET_N, RESET_CLIPS, RESET_SEED, TABLE_SEED = 64, 9, 61, 62
PROB = [0.2, 0.0, 0.1, 0.15, 0.05, 0.0, 0.2, 0.2, 0.1]
DT = 1.0 / 30.0
MAX_LEN = 300


def inputs(N, seed=0):
    """Seeded 52-body simulator rows: some envs fall (a non-contact body pressed and one low), some sit at progress <= 1, some at the
    episode's end."""
    g = torch.Generator().manual_seed(seed)
    unit = lambda q: q / q.norm(dim=-1, keepdim=True)
    bs = torch.zeros(N, BODIES, 13)
    bs[..., 0:3] = torch.randn(N, BODIES, 3, generator=g) * 0.4 + torch.tensor([0.0, 0.0, 0.9])
    bs[::5, 30:, 2] = 0.05                                   # low hands: fall by height
    bs[..., 3:7] = unit(torch.randn(N, BODIES, 4, generator=g))
    bs[..., 7:13] = torch.randn(N, BODIES, 6, generator=g)
    prev_root = bs[:, 0, 0:3] - torch.randn(N, 3, generator=g) * 0.04
    tar_speed = torch.rand(N, generator=g) * 4 + 0.5
    contact = torch.zeros(N, BODIES, 3)
    contact[::2] = torch.randn((N + 1) // 2, BODIES, 3, generator=g) * (torch.rand((N + 1) // 2, BODIES, 1, generator=g) < 0.1) * 60
    progress = torch.randint(0, 310, (N,), generator=g)
    progress[::11] = 1
    progress[3::13] = MAX_LEN - 1
    term_h = torch.full((BODIES,), 0.15)
    bs[2::17, :, 2] = 1.0                                    # only body 40 low and pressed: its contact bit decides the fall
    bs[2::17, 40, 2] = 0.05
    contact[2::17] = 0.0
    contact[2::17, 40, 2] = 5.0
    return dict(body_state=bs, prev_root_pos=prev_root, tar_speed=tar_speed, contact_forces=contact, progress_buf=progress, termination_heights=term_h)


def main():
    import importlib
    from oracle.refshim.load_reference import load_reference
    ref = load_reference()
    ref.flags.follow = False               # set by run_hydra.py's flag parser in a real run
    speed = importlib.import_module("env.tasks.humanoid_speed")
    N = 211
    z = inputs(N)
    bs, root = z["body_state"], z["body_state"][:, 0]
    empty = torch.zeros(N, 0)
    out = {"num_envs": np.int64(N)}
    out["self_obs"] = ref.humanoid.compute_humanoid_observations_smpl_max(bs[..., 0:3], bs[..., 3:7], bs[..., 7:10], bs[..., 10:13], empty, empty,
                                                                          True, True, False, False, False)
    out["base_removed"] = ref.humanoid.remove_base_rot(root[:, 3:7])
    out["speed_obs"] = speed.compute_speed_observations(root, z["tar_speed"])
    out["speed_reward"] = speed.compute_speed_reward(root[:, 0:3], z["prev_root_pos"], root[:, 3:7], z["tar_speed"], DT)
    rs, tm = ref.humanoid.compute_humanoid_reset(torch.zeros(N, dtype=torch.long), z["progress_buf"], z["contact_forces"], torch.tensor(CONTACT_IDS),
                                                 bs[..., 0:3], MAX_LEN, True, z["termination_heights"])
    out["reset"], out["terminate"] = rs, tm
    rs, tm = ref.humanoid.compute_humanoid_reset(torch.zeros(N, dtype=torch.long), z["progress_buf"], z["contact_forces"],
                                                 torch.tensor(CONTACT_IDS_HI), bs[..., 0:3], MAX_LEN, True, z["termination_heights"])
    out["reset_hi"], out["terminate_hi"] = rs, tm
    out.update(reset_fixture(speed.HumanoidSpeed))
    np.savez_compressed(os.path.join(HERE, "smplx_speed.npz"), **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
    print({k: getattr(v, "shape", None) for k, v in out.items()}, "terminated (hi):", int(tm.sum()), "draws:", str(out["r_draws"]))


def reset_fixture(HumanoidSpeed):
    """HumanoidSpeed._reset_ref_state_init + _reset_task on a 52-body stand-in, StateInit Random, has_upright_start False.  Keys r_*."""
    from phc.utils.motion_lib_smpl import MotionLibSMPL
    from tests import smplx_speed_oracle as so
    from tests import ztask_reset_oracle as zo
    speed_mod = sys.modules[HumanoidSpeed.__module__]
    if not hasattr(speed_mod, "quat_apply"):   # isaacgym.torch_utils.quat_apply, which the Isaac Gym stand-in does not define
        from oracle.terrain_oracle import quat_apply
        speed_mod.quat_apply = quat_apply
    N = RESET_N
    tb = so.tables(RESET_CLIPS, seed=TABLE_SEED)
    betas = torch.linspace(-1.0, 1.0, 10)
    lib = MotionLibSMPL.__new__(MotionLibSMPL)
    for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs"):
        setattr(lib, k, getattr(tb, k))
    lib._motion_aa, lib._motion_lengths, lib._motion_num_frames, lib._motion_dt = tb.motion_aa, tb.lengths, tb.num_frames, tb.dt
    lib.length_starts, lib._motion_bodies, lib._motion_limb_weights = tb.length_starts, torch.zeros(RESET_CLIPS, 17), torch.zeros(RESET_CLIPS, 10)
    lib.num_bodies, lib._device = BODIES, "cpu"
    lib._sampling_batch_prob = torch.tensor(PROB)

    class Task(HumanoidSpeed):
        def __init__(self):
            pass

    t = Task()
    t.device, t.humanoid_type, t.dt = "cpu", "smplx", zo.DT
    t._state_init = next(c for c in HumanoidSpeed.__mro__ if c.__name__ == "HumanoidAMP").StateInit.Random
    t._motion_lib, t.ref_motion_cache = lib, {}
    t.smpl_parser_n = t.smpl_parser_m = t.smpl_parser_f = so.Parser72(zo.StandInParser())
    t.humanoid_shapes = torch.cat([torch.ones(N, 1), betas.expand(N, 10)], dim=-1)          # gender 1, one shape
    t.humanoid_limb_and_weights = torch.zeros(N, 10)
    t._humanoid_root_states = torch.zeros(N, 13)
    t._dof_pos, t._dof_vel = torch.zeros(N, DOFS), torch.zeros(N, DOFS)
    rb = torch.zeros(N, BODIES, 13)
    t._rigid_body_pos, t._rigid_body_rot, t._rigid_body_vel, t._rigid_body_ang_vel = rb[..., 0:3], rb[..., 3:7], rb[..., 7:10], rb[..., 10:13]
    t._motion_start_times, t._sampled_motion_ids = torch.zeros(N), torch.zeros(N, dtype=torch.long)
    t._body_names, t._has_upright_start, t.power_acc = ["body%d" % i for i in range(BODIES)], False, torch.ones(N, 2)
    t.progress_buf = torch.randint(0, 50, (N,), generator=torch.Generator().manual_seed(RESET_SEED))
    t._tar_speed, t._speed_change_steps = torch.ones(N), torch.zeros(N, dtype=torch.long)
    t._tar_speed_min, t._tar_speed_max = zo.SPEED["tar_speed_min"], zo.SPEED["tar_speed_max"]
    t._speed_change_steps_min, t._speed_change_steps_max = zo.SPEED["steps_min"], zo.SPEED["steps_max"]
    env_ids = torch.from_numpy(np.flatnonzero(np.random.default_rng(RESET_SEED).random(N) < 0.6)).long()
    rec = []
    multinomial0, rand0, randint0 = torch.multinomial, torch.rand, torch.randint

    def wrap(name, fn):
        def f(*a, **k):
            res = fn(*a, **k)
            rec.append((name, res.clone()))
            return res
        return f

    torch.manual_seed(RESET_SEED)
    torch.multinomial, torch.rand, torch.randint = wrap("multinomial", multinomial0), wrap("rand", rand0), wrap("randint", randint0)
    try:
        t._reset_ref_state_init(env_ids)
        t._reset_task(env_ids)
    finally:
        torch.multinomial, torch.rand, torch.randint = multinomial0, rand0, randint0
    out = {"r_env_ids": env_ids.numpy(), "r_progress": t.progress_buf.numpy(), "r_draws": np.array(" ".join(n for n, _ in rec)),
           "r_root_states": t._humanoid_root_states.numpy(), "r_dof_pos": t._dof_pos.numpy(), "r_dof_vel": t._dof_vel.numpy(),
           "r_body_state": rb.numpy(), "r_start_times": t._motion_start_times.numpy(), "r_motion_ids": t._sampled_motion_ids.numpy(),
           "r_power_acc": t.power_acc.numpy(), "r_tar_speed": t._tar_speed.numpy(), "r_change_steps": t._speed_change_steps.numpy(),
           "r_prob": np.array(PROB, dtype=np.float32)}
    for i, (_, v) in enumerate(rec):
        out[f"r_draw{i}"] = v.numpy()
    return out


if __name__ == "__main__":
    main()
