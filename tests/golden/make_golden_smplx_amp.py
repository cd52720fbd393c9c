"""Fixture for the PULSE-X AMP rows (HumanoidSpeedZ with robot=smplx_humanoid, env_pulsex_amp.yaml): outputs of the UNMODIFIED
reference's build_amp_observations_smpl (humanoid_amp.py:925-969) with the SMPL-X dof_subset (joints 0..50 without L_Toe and R_Toe,
humanoid.py:404-421), key bodies R_Ankle, L_Ankle, R_Wrist, L_Wrist = (7, 3, 36, 17) and upright False, on seeded 52-body states,
with and without the root height; and of its _init_amp_obs_ref (:535-563) and build_amp_obs_demo_steps (:232-251) on a 52-body
stand-in over the tables of `tests.smplx_speed_oracle.tables`.

  * Root rotations are random unit quaternions, far from upright, so remove_base_rot changes every row's heading.
  * The dofs of every joint are non-zero, the dropped toes' included, so a column they leaked into would show.
  * Only the 466-float rows are stored: the generator checks that the reference's 465-float rows (ampRootHeightObs False) are the
    466-float ones without their first column, so a test takes those as row[..., 1:].  This keeps the fixture small.
  * The stand-in subclasses HumanoidSpeed without its constructor and holds an un-initialised reference MotionLibSMPL with the tables,
    as tests/golden/make_golden_smplx_speed.py does; only body indices enter (no smpl_sim name list).

  python tests/golden/make_golden_smplx_amp.py     (needs the reference tree; writes tests/golden/smplx_amp.npz)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

BODIES, DOFS = 52, 153
KEY_BODY_IDS = [7, 3, 36, 17]
DOF_SUBSET = [k for k in range(DOFS) if (k // 3) not in (3, 7)]
N_STATE, STATE_SEED = 24, 71
CLIPS, TABLE_SEED, N_REF, REF_SEED, STEPS = 7, 72, 5, 73, 10
DT = float(np.float32(1.0 / 60.0) * 2)


def state_inputs(n=N_STATE, seed=STATE_SEED):
    """Seeded 52-body simulator rows [n, 52, 13] and dof positions / velocities [n, 153]."""
    g = torch.Generator().manual_seed(seed)
    bs = torch.zeros(n, BODIES, 13)
    bs[..., 0:3] = torch.randn(n, BODIES, 3, generator=g) * 0.4 + torch.tensor([0.0, 0.0, 0.9])
    q = torch.randn(n, BODIES, 4, generator=g)
    bs[..., 3:7] = q / q.norm(dim=-1, keepdim=True)
    bs[..., 7:13] = torch.randn(n, BODIES, 6, generator=g)
    dof_pos = torch.randn(n, DOFS, generator=g) * 0.8
    dof_pos[3::11, 9:12] = 1e-7                              # near-zero rotations: the exponential map's identity branch
    dof_vel = torch.randn(n, DOFS, generator=g)
    return bs, dof_pos, dof_vel


def ref_inputs(n=N_REF, seed=REF_SEED):
    """Clips and start times of the motion rows: (motion ids [n], t0 [n]) within each clip, some before dt * (STEPS - 1)."""
    from tests import smplx_speed_oracle as so
    tb = so.tables(CLIPS, seed=TABLE_SEED)
    g = torch.Generator().manual_seed(seed)
    mids = torch.randint(0, CLIPS, (n,), generator=g)
    t0 = torch.rand(n, generator=g) * tb.lengths[mids]
    t0[::5] = 0.05
    return tb, mids, t0


def main():
    import importlib
    from oracle.refshim.load_reference import load_reference
    ref = load_reference()
    ref.flags.follow = False
    amp = importlib.import_module("env.tasks.humanoid_amp")
    speed = importlib.import_module("env.tasks.humanoid_speed")
    bs, dof_pos, dof_vel = state_inputs()
    n = bs.shape[0]
    subset = torch.tensor(DOF_SUBSET)
    out = {"num_envs": np.int64(n), "key_body_ids": np.array(KEY_BODY_IDS), "dof_subset": subset.numpy()}
    rows = {h: amp.build_amp_observations_smpl(bs[:, 0, 0:3], bs[:, 0, 3:7], bs[:, 0, 7:10], bs[:, 0, 10:13], dof_pos, dof_vel,
                                               bs[:, KEY_BODY_IDS, 0:3], torch.zeros(n, 0), torch.zeros(n, 0), subset, True, h, True, False,
                                               False, False) for h in (True, False)}
    assert rows[True].shape[1] == 466 and torch.equal(rows[False], rows[True][:, 1:])
    out["state_amp"] = rows[True]
    out.update(motion_fixture(speed.HumanoidSpeed))
    np.savez_compressed(os.path.join(HERE, "smplx_amp.npz"), **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
    print({k: getattr(v, "shape", None) for k, v in out.items()})


def motion_fixture(HumanoidSpeed):
    """_init_amp_obs_ref (rows t0 - k dt, k = 1 .. STEPS - 1) and build_amp_obs_demo_steps (k = 0 .. STEPS - 1) of the stand-in, with and
    without the root height (checked to differ only by the first column).  Keys init, demo: the 466-float rows [n, rows, 466]."""
    from phc.utils.motion_lib_smpl import MotionLibSMPL
    tb, mids, t0 = ref_inputs()
    n = mids.shape[0]
    lib = MotionLibSMPL.__new__(MotionLibSMPL)
    for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs"):
        setattr(lib, k, getattr(tb, k))
    lib._motion_aa, lib._motion_lengths, lib._motion_num_frames, lib._motion_dt = tb.motion_aa, tb.lengths, tb.num_frames, tb.dt
    lib.length_starts, lib._motion_bodies, lib._motion_limb_weights = tb.length_starts, torch.zeros(CLIPS, 17), torch.zeros(CLIPS, 10)
    lib.num_bodies, lib._device = BODIES, "cpu"

    class Task(HumanoidSpeed):
        def __init__(self):
            pass

    t = Task()
    t.device, t.humanoid_type, t.dt, t.amp_obs_v = "cpu", "smplx", DT, 1
    t._motion_lib, t.ref_motion_cache = lib, {}
    t._key_body_ids, t.dof_subset, t._has_dof_subset = torch.tensor(KEY_BODY_IDS), torch.tensor(DOF_SUBSET), True
    t._local_root_obs, t._has_shape_obs_disc, t._has_limb_weight_obs_disc, t._has_upright_start = True, False, False, False
    t._num_amp_obs_steps = STEPS
    out = {"ref_motion_ids": mids.numpy(), "ref_t0": t0.numpy()}
    got = {}
    for h in (True, False):
        t._amp_root_height_obs = h
        width = 466 if h else 465
        t._hist_amp_obs_buf = torch.zeros(n, STEPS - 1, width)
        t.ref_motion_cache = {}
        t._init_amp_obs_ref(torch.arange(n), mids, t0)
        got[h] = (t._hist_amp_obs_buf.clone(), t.build_amp_obs_demo_steps(mids, t0, STEPS).view(n, STEPS, width))
    for a, b in zip(got[False], got[True]):
        assert torch.equal(a, b[..., 1:])
    out["init"], out["demo"] = got[True]
    return out


if __name__ == "__main__":
    main()
