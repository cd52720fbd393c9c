"""The reset kernels element-wise against the float64 references of tests/reset_fp64.py, with every Philox word regenerated on the host:
`pulse_reset_ref_state`, `pulse_reset_getup` + `pulse_getup_amp_init`, `pulse_reset_ztask` (reach, speed, strike) with
`pulse_ztask_reset_task`, `pulse_reset_ztask_smplx` (52 bodies) and `pulse_reset_terrain`, on clips at 24 to 120 fps (2-frame clips
included).  Each case runs twice, once with the host-regenerated draws injected and once with the kernel's own Philox draws: both
runs must agree bit for bit, and both pass the links.  `-s` prints every margin."""
import numpy as np
import pytest
import torch

from tests import reset_fp64 as rf
from tests.helpers import clip_rates, exact_tables

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
RATES = [24.0, 25.0, 29.97, 30.0, 50.0, 60.0, 120.0]
KEYS = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "lengths", "num_frames", "dt", "length_starts")
CLIPS = 29
SEED, OFF = 4242, 9
STEPS = 5
SIZES = [1, 257, 2051, 16384]


@pytest.fixture(scope="module")
def rep():
    r = rf.Report("reset kernels vs float64 references")
    yield r
    print("\n" + r.text())


def _tables(smplx=False):
    if smplx:
        from tests.smplx_speed_oracle import tables
        tb = tables(CLIPS, seed=6)
        rates = clip_rates(RATES, CLIPS)
        t = {k: getattr(tb, k).clone() for k in KEYS if k not in ("lengths", "dt")}
        t["num_frames"][1] = 2
        t.update(dt=(1.0 / rates).float(), lengths=((t["num_frames"] - 1).double() * (1.0 / rates)).float())
        t["length_starts"] = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(t["num_frames"], 0)[:-1]])
        F = int(t["num_frames"].sum())
        for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs"):
            t[k] = t[k][:F].contiguous()
    else:
        tb = exact_tables(CLIPS, seed=6, fps=RATES)
        t = {k: getattr(tb, k).clone() for k in KEYS + ("motion_aa",)}
    s, nf = int(t["length_starts"][4]), int(t["num_frames"][4])
    t["lrs"][s:s + nf, 1:5] = torch.tensor([0.0, 0.0, 0.0, 1.0])      # identity joints: the exp-map zero and the identity branch
    return t


@pytest.fixture(scope="module")
def smpl():
    from pulse_b200.motion_lib import MotionLibB200
    t = _tables()
    ml = MotionLibB200.from_tables(dict(t), device=DEV)
    p = torch.rand(CLIPS, generator=torch.Generator().manual_seed(4))
    p[[2, 9, CLIPS - 1]] = 0.0                        # a trailing zero-weight clip: the pick's nextafter clamp
    ml._sampling_batch_prob = (p / p.sum()).to(DEV)
    floor = (-0.9 + 0.1 * torch.rand(t["gts"].shape[0], generator=torch.Generator().manual_seed(5))).to(DEV)
    return t, ml, floor


@pytest.fixture(scope="module")
def smplx():
    from pulse_b200.motion_lib import MotionLibB200
    t = _tables(smplx=True)
    ml = MotionLibB200.from_tables(dict(t), device=DEV)
    ml._sampling_batch_prob = torch.full((CLIPS,), 1.0 / CLIPS, device=DEV)
    floor = (-0.9 + 0.1 * torch.rand(t["gts"].shape[0], generator=torch.Generator().manual_seed(5))).to(DEV)
    return t, ml, floor


def _state(n, B, D, seed, width=196):
    g = torch.Generator().manual_seed(seed)
    d = {"root_all": torch.randn(n, 2, 13, generator=g), "dof_state": torch.randn(n, D + 3, 2, generator=g),
         "body": torch.randn(n, B + 2, 13, generator=g), "contact": torch.randn(n, B + 2, 3, generator=g),
         "sampled_motion_ids": torch.randint(0, CLIPS, (n,), generator=g), "motion_start_times": torch.rand(n, generator=g),
         "progress_buf": torch.randint(0, 300, (n,), generator=g), "reset_buf": torch.zeros(n, dtype=torch.int64),
         "terminate_buf": (torch.rand(n, generator=g) < 0.3).long(), "amp": torch.randn(n, STEPS, width, generator=g)}
    return {k: v.to(DEV) for k, v in d.items()}


def _ids(n, frac, seed):
    ids = (torch.rand(n, generator=torch.Generator().manual_seed(seed)) < frac).nonzero().flatten()
    return ids if ids.numel() else torch.tensor([n // 2])


def _bad_list(n):
    """Unsorted, duplicate and out-of-range ids: an id outside [0, N) or not above its predecessor is skipped."""
    raw = [5, 3, 3, 7, -1, n + 4, 9, 9, 12, 30, 31, 29, n - 1]
    raw = [x for x in raw if x < n or x == n + 4] if n > 31 else [0, 0, n, n - 1]
    out, prev = [], None
    for x in raw:
        if 0 <= x < n and (prev is None or prev < x):
            out.append(x)
        prev = x
    return torch.tensor(raw, dtype=torch.int64), torch.tensor(out, dtype=torch.int64)


def _same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}: injected and Philox runs differ in {k}"


def _untouched(d, d0, ids, n, keys=("root_all", "body", "dof_state", "amp", "contact", "sampled_motion_ids", "motion_start_times", "progress_buf",
                                     "reset_buf", "terminate_buf")):
    keep = torch.ones(n, dtype=torch.bool, device=DEV)
    keep[ids.to(DEV)] = False
    for k in keys:
        assert torch.equal(d[k][keep], d0[k][keep]), k


# ---------------------------------------------------------------------------------------------------------------- latent tasks
def _ztask_run(r, d, kind, B, D, mode_ids, draws, amp):
    kw = dict(root_states=d["root_all"][:, 0], dof_pos=d["dof_state"][:, :D, 0], dof_vel=d["dof_state"][:, :D, 1], rigid_body_state=d["body"],
              progress_buf=d["progress_buf"], sampled_motion_ids=d["sampled_motion_ids"], motion_start_times=d["motion_start_times"],
              terminate_buf=d["terminate_buf"], contact_forces=d["contact"], amp_obs_buf=d["amp"] if amp else None,
              seed=SEED, offset=OFF)
    if mode_ids is None:
        kw["reset_buf"] = d["reset_buf"]
    else:
        kw["env_ids"] = mode_ids.to(DEV)
    if kind == "strike":
        kw["target_states"] = d["root_all"][:, 1]
    if draws is not None:
        kw.update(motion_u=draws["motion_u"].to(DEV), phase=draws["phase"].to(DEV))
        if kind == "strike":
            kw["strike_u"] = draws["strike_u"].to(DEV).contiguous()
    return r.reset_envs(**kw)


def _check_ztask(rep, tag, t, ml, floor, kind, upright, d, ids, B, D, amp, width, init="Random"):
    n = d["progress_buf"].shape[0]
    idc = ids.cpu()
    dr = rf.ztask_draws(SEED, idc, OFF)
    mids = rf.pick_motion_ref(ml.sampling_cdf(), dr["motion_u"])
    rf.check_exact(rep, f"{tag} draws clip", d["sampled_motion_ids"][ids].cpu(), mids)
    t0 = rf.start_time_ref(dr["phase"], t["lengths"][mids]) if init == "Random" else torch.zeros(len(idc))
    rf.check_exact(rep, f"{tag} draws start time", d["motion_start_times"][ids].cpu(), t0)
    pose = {"reach": rf.POSE_ROOT_XY_ZERO, "strike": rf.POSE_ROOT_XY_ZERO, "speed": rf.POSE_FACE_X}[kind]
    td = {k: v.to(DEV) for k, v in t.items()}
    ref = rf.reset_state_ref(td, mids.to(DEV), t0.to(DEV), floor, pose, upright)
    got = {"body": d["body"][ids, :B], "root": d["root_all"][ids, 0], "dof_pos": d["dof_state"][ids, :D, 0], "dof_vel": d["dof_state"][ids, :D, 1]}
    rf.check_state(rep, tag, got, ref)
    rf.check_exact(rep, f"{tag} counters", torch.stack([d["progress_buf"][ids], d["reset_buf"][ids], d["terminate_buf"][ids]]).cpu(),
                   torch.zeros(3, len(idc), dtype=torch.int64))
    rf.check_exact(rep, f"{tag} contact forces", d["contact"][ids].cpu(), torch.zeros(len(idc), B + 2, 3))
    if kind == "strike":
        s = rf.strike_ref(dr["strike_u"].to(DEV), torch.zeros(len(idc), 2, device=DEV), 0.5, 1.5, 0.5, 10.0)
        tg = d["root_all"][ids, 1]
        rf.check(rep, f"{tag} strike target xy", tg[:, :2], *s["xy"])
        rf.check(rep, f"{tag} strike target yaw", tg[:, 5:7], *s["zw"])
        rf.check_exact(rep, f"{tag} strike target rest", torch.cat([tg[:, 2:5], tg[:, 7:]], 1).cpu(),
                       torch.tensor([0.9, 0, 0] + [0] * 6).expand(len(idc), 9))
    if amp:
        a = d["amp"][ids]
        rf.check_amp(rep, f"{tag} row 0", a[:, 0], rf.state_amp_ref(got["body"], got["dof_pos"], got["dof_vel"], upright))
        times = rf.history_times(t0, float(np.float32(1.0 / 60.0) * 2), STEPS)
        for k in range(1, STEPS):
            rf.check_amp(rep, f"{tag} row {k}", a[:, k], rf.motion_amp_ref(rf.motion_ref(td, mids.to(DEV), times[:, k].to(DEV)), upright))


ZCASES = [("reach", True, "Random"), ("speed", False, "Random"), ("strike", True, "Random"), ("speed", True, "Start")]


def _mode(n, frac):
    """Mask and list mode alternate over the sizes, so every size and fraction meets both across the two fractions."""
    return ("mask", "list")[(SIZES.index(n) + (frac == 1.0)) % 2]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("frac", [0.05, 1.0])
@pytest.mark.parametrize("kind,upright,init", ZCASES)
def test_ztask_reset(rep, smpl, n, frac, kind, upright, init):
    from pulse_b200.ztask_reset import ZTaskResetB200
    t, ml, floor = smpl
    r = ZTaskResetB200(kind, ml, floor, upright=upright, state_init=init)
    ids = _ids(n, frac, n + 1)
    mode = _mode(n, frac)
    runs = []
    for inject in (True, False):
        d = _state(n, 24, 69, seed=n, width=195)
        d0 = {k: v.clone() for k, v in d.items()}
        dr = rf.ztask_draws(SEED, torch.arange(n), OFF) if inject else None
        if mode == "mask":
            d["reset_buf"][ids.to(DEV)] = 1
        ws = _ztask_run(r, d, kind, 24, 69, None if mode == "mask" else ids, dr, True)
        torch.cuda.synchronize()
        assert int(ws["count"].item()) == ids.numel() and torch.equal(ws["env_list"][:ids.numel()].cpu(), ids)
        if kind != "strike":
            chg = torch.zeros(n, dtype=torch.int64, device=DEV)
            tar = torch.zeros(n, 3, device=DEV) if kind == "reach" else torch.zeros(n, device=DEV)
            td = rf.task_draws(SEED, torch.arange(n), OFF, 100, 200)
            kw = dict(rand=(td["rand"] if kind == "reach" else td["rand"][:, 0].contiguous()).to(DEV), steps=td["steps"].to(DEV)) if inject else {}
            r.reset_task(progress_buf=d["progress_buf"], change_steps=chg, seed=SEED, offset=OFF,
                         **({"tar_pos": tar} if kind == "reach" else {"tar_speed": tar}), **kw)
            d["tar"], d["chg"] = tar, chg
        torch.cuda.synchronize()
        tag = f"ztask {kind}{'' if upright else ' non-upright'} {init} n={n} {frac} {mode}{' injected' if inject else ''}"
        _check_ztask(rep, tag, t, ml, floor, kind, upright, d, ids.to(DEV), 24, 69, True, 195, init)
        if kind != "strike":
            tdr = rf.task_draws(SEED, ids, OFF, 100, 200)
            tr = rf.task_ref(kind, tdr["rand"], tdr["steps"], torch.zeros(len(ids), dtype=torch.int64), 1.0, 0.5, 1.5, 0.0, 5.0)
            rf.check_exact(rep, f"{tag} task change steps", d["chg"][ids.to(DEV)].cpu(), tr["change_steps"])
            rf.check(rep, f"{tag} task target", d["tar"][ids.to(DEV)].cpu(), *tr["target"])
        _untouched(d, d0, ids, n)
        runs.append(d)
    _same(runs[0], runs[1], f"ztask {kind} n={n}")


def test_ztask_reset_edge_draws(rep, smpl):
    """Injected edge draws: phase 0 and one ulp below 1 (the largest u01); clip uniforms 0 (the first clip with weight), one ulp below
    1 and 1.0.  At u = 1.0, u * total equals total: the nextafter clamp of pick_motion keeps the pick on the last clip with weight,
    where without it the search would run past to the trailing zero-weight clip."""
    from pulse_b200.ztask_reset import ZTaskResetB200
    t, ml, floor = smpl
    n = 257
    r = ZTaskResetB200("reach", ml, floor, amp_root_height_obs=True)
    top = float(np.float32(1 - 2 ** -24))
    ph = torch.tensor([0.0, top] * (n // 2) + [top])
    mu = torch.tensor([1.0, 0.0, top, 0.5] * (n // 4) + [1.0] * (n % 4))
    d = _state(n, 24, 69, seed=8)
    ids = torch.arange(n)
    r.reset_envs(root_states=d["root_all"][:, 0], dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1], rigid_body_state=d["body"],
                 progress_buf=d["progress_buf"], sampled_motion_ids=d["sampled_motion_ids"], motion_start_times=d["motion_start_times"],
                 env_ids=ids.to(DEV), terminate_buf=d["terminate_buf"], contact_forces=d["contact"], amp_obs_buf=d["amp"],
                 motion_u=mu.to(DEV), phase=ph.to(DEV))
    torch.cuda.synchronize()
    mids = rf.pick_motion_ref(ml.sampling_cdf(), mu)
    assert float(ml._sampling_batch_prob[CLIPS - 1]) == 0.0 and float(ml._sampling_batch_prob[CLIPS - 2]) > 0.0
    assert int(mids[0]) == CLIPS - 2 and int(mids[1]) == 0 and int(mids[2]) == CLIPS - 2
    rf.check_exact(rep, "ztask edges clip", d["sampled_motion_ids"].cpu(), mids)
    t0 = rf.start_time_ref(ph, t["lengths"][mids])
    rf.check_exact(rep, "ztask edges start time", d["motion_start_times"].cpu(), t0)
    td = {k: v.to(DEV) for k, v in t.items()}
    ref = rf.reset_state_ref(td, mids.to(DEV), t0.to(DEV), floor, rf.POSE_ROOT_XY_ZERO, True)
    got = {"body": d["body"][:, :24], "root": d["root_all"][:, 0], "dof_pos": d["dof_state"][:, :69, 0], "dof_vel": d["dof_state"][:, :69, 1]}
    rf.check_state(rep, "ztask edges", got, ref)
    rf.check_amp(rep, "ztask edges row 0 (196)", d["amp"][:, 0], rf.state_amp_ref(got["body"], got["dof_pos"], got["dof_vel"], True))
    times = rf.history_times(t0, float(np.float32(1.0 / 60.0) * 2), STEPS)
    for k in range(1, STEPS):
        rf.check_amp(rep, f"ztask edges row {k} (196)", d["amp"][:, k], rf.motion_amp_ref(rf.motion_ref(td, mids.to(DEV), times[:, k].to(DEV)), True))


def _smplx_run(rep, tag, smplx, d, mode_ids, inject):
    from pulse_b200 import _lib
    from pulse_b200.ztask_reset import ZTaskResetB200
    t, ml, floor = smplx
    B, D = _lib.SMPLX_BODIES, _lib.SMPLX_DOF
    n = d["progress_buf"].shape[0]
    r = ZTaskResetB200("speed", ml, floor, upright=False)
    ws = _ztask_run(r, d, "speed", B, D, mode_ids, rf.ztask_draws(SEED, torch.arange(n), OFF) if inject else None, False)
    torch.cuda.synchronize()
    return ws, lambda ids: _check_ztask(rep, tag, t, ml, floor, "speed", False, d, ids.to(DEV), B, D, False, 0)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("frac", [0.05, 1.0])
def test_smplx_reset(rep, smplx, n, frac):
    """pulse_reset_ztask_smplx: 52 bodies, lane l holding bodies l and l + 32, FACE_X of the non-upright heading."""
    from pulse_b200 import _lib
    ids = _ids(n, frac, n + 2)
    mode = _mode(n, frac)
    runs = []
    for inject in (True, False):
        d = _state(n, _lib.SMPLX_BODIES, _lib.SMPLX_DOF, seed=n + 1)
        d0 = {k: v.clone() for k, v in d.items()}
        if mode == "mask":
            d["reset_buf"][ids.to(DEV)] = 1
        ws, check = _smplx_run(rep, f"smplx n={n} {frac} {mode}{' injected' if inject else ''}", smplx, d, None if mode == "mask" else ids, inject)
        assert int(ws["count"].item()) == ids.numel() and torch.equal(ws["env_list"][:ids.numel()].cpu(), ids)
        check(ids)
        _untouched(d, d0, ids, n)
        runs.append(d)
    _same(runs[0], runs[1], f"smplx n={n}")


# ---------------------------------------------------------------------------------------------------------------- terrain
@pytest.fixture(scope="module")
def terrain():
    from pulse_b200.terrain import TerrainB200, center_height_points
    g = torch.Generator().manual_seed(6)
    hf = torch.randint(-200, 200, (120, 130), generator=g, dtype=torch.int16)
    cells = torch.randint(5, 110, (997, 2), generator=g)
    cx, cy = cells[:, 0].float() * 0.1, cells[:, 1].float() * 0.1
    return hf, cx, cy, center_height_points().float(), TerrainB200(hf, device=DEV)


def _terrain_run(rep, tag, smpl, terrain, d, mode_ids, upright, inject):
    """pulse_reset_terrain and then pulse_traj_reset_list from the roots it wrote, with the host-regenerated draws injected or the
    kernels' own Philox draws.  Returns the workspace and a check of the listed envs against the references."""
    from pulse_b200.terrain import PedestrianTerrainTaskB200
    from pulse_b200.terrain_reset import TerrainResetB200
    t, ml, floor = smpl
    hf, cx, cy, pts, tr = terrain
    n = d["progress_buf"].shape[0]
    r = TerrainResetB200(ml, floor, tr, cx, cy, upright=upright)
    task = PedestrianTerrainTaskB200(n, device=DEV, terrain=tr, dt=1.0 / 30.0, seed=SEED)
    full = rf.ztask_draws(SEED, torch.arange(n), OFF)
    kw = dict(motion_u=full["motion_u"].to(DEV), phase=full["phase"].to(DEV), loc_ids=rf.terrain_loc(full["r0"], len(cx)).to(DEV)) if inject else {}
    kw.update(env_ids=mode_ids.to(DEV)) if mode_ids is not None else kw.update(reset_buf=d["reset_buf"])
    ws = r.reset_envs(root_states=d["root_all"][:, 0], dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1],
                      rigid_body_state=d["body"], progress_buf=d["progress_buf"], sampled_motion_ids=d["sampled_motion_ids"],
                      motion_start_times=d["motion_start_times"], terminate_buf=d["terminate_buf"], contact_forces=d["contact"],
                      amp_obs_buf=d["amp"], seed=SEED, offset=OFF, **kw)
    rand = rf.traj_draws(SEED, torch.arange(n), OFF).to(DEV) if inject else None
    r.reset_task(task, d["root_all"][:, 0], rand=rand, seed=SEED, offset=OFF)
    torch.cuda.synchronize()
    d["traj"] = task.traj_verts
    params = (task.dtheta_max * task.traj_dt, task.accel_max * task.traj_dt, task.traj_dt, task.speed_min, task.speed_max, task.sharp_turn_prob)

    def check(ids):
        idd = ids.to(DEV)
        dr = rf.ztask_draws(SEED, ids, OFF)
        loc = rf.terrain_loc(dr["r0"], len(cx))
        rf.check_exact(rep, f"{tag} location", ws["loc_ids"][idd].cpu(), loc)
        mids = rf.pick_motion_ref(ml.sampling_cdf(), dr["motion_u"])
        rf.check_exact(rep, f"{tag} draws clip", d["sampled_motion_ids"][idd].cpu(), mids)
        t0 = rf.start_time_ref(dr["phase"], t["lengths"][mids])
        rf.check_exact(rep, f"{tag} draws start time", d["motion_start_times"][idd].cpu(), t0)
        td = {k: v.to(DEV) for k, v in t.items()}
        ref = rf.reset_state_ref(td, mids.to(DEV), t0.to(DEV), floor, rf.POSE_AS_IS, upright)
        got = {"body": d["body"][idd, :24], "root": d["root_all"][idd, 0], "dof_pos": d["dof_state"][idd, :69, 0], "dof_vel": d["dof_state"][idd, :69, 1]}
        sp = rf.spawn_ref(ref, loc.to(DEV), cx.to(DEV), cy.to(DEV), hf.to(DEV), 0.1, 0.005, pts, upright, got["root"][:, 3:7])
        ref["body_pos"], ref["root_pos"] = sp["body_pos"], sp["root_pos"]
        rf.limit_share(rep, f"{tag} cell edge", sp["edge"], amb_max=rf.EDGE_MAX)
        rf.check_state(rep, tag, got, ref)
        rf.check_amp(rep, f"{tag} row 0", d["amp"][idd, 0], rf.state_amp_ref(got["body"], got["dof_pos"], got["dof_vel"], upright))
        times = rf.history_times(t0, float(np.float32(1.0 / 60.0) * 2), STEPS)
        for k in range(1, STEPS):
            rf.check_amp(rep, f"{tag} row {k}", d["amp"][idd, k], rf.motion_amp_ref(rf.motion_ref(td, mids.to(DEV), times[:, k].to(DEV)), upright))
        start = got["root"][:, :2]
        rf.check_traj(rep, tag, d["traj"][idd], start, rf.traj_ref(start, rf.traj_draws(SEED, ids, OFF), *params))
        keep = torch.ones(n, dtype=torch.bool, device=DEV)
        keep[idd] = False
        assert not d["traj"][keep].any(), "waypoints of an env that was not reset"

    return ws, check


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("frac", [0.05, 1.0])
@pytest.mark.parametrize("upright", [True, False])
def test_terrain_reset(rep, smpl, terrain, n, frac, upright):
    ids = _ids(n, frac, n + 3)
    mode = _mode(n, frac)
    runs = []
    for inject in (True, False):
        d = _state(n, 24, 69, seed=n + 2)
        d0 = {k: v.clone() for k, v in d.items()}
        if mode == "mask":
            d["reset_buf"][ids.to(DEV)] = 1
        tag = f"terrain{'' if upright else ' non-upright'} n={n} {frac} {mode}{' injected' if inject else ''}"
        ws, check = _terrain_run(rep, tag, smpl, terrain, d, None if mode == "mask" else ids, upright, inject)
        assert int(ws["count"].item()) == ids.numel() and torch.equal(ws["env_list"][:ids.numel()].cpu(), ids)
        check(ids)
        _untouched(d, d0, ids, n)
        runs.append(d)
    _same(runs[0], runs[1], f"terrain n={n}")


@pytest.mark.parametrize("kind", ["reach", "strike", "smplx", "terrain"])
def test_reset_skips_bad_ids(rep, smpl, smplx, terrain, kind):
    """The resets built on reset_warps.cuh skip an id outside [0, N) or not above its predecessor: unsorted, duplicate and
    out-of-range ids leave each listed env written once and every other env untouched."""
    from pulse_b200 import _lib
    from pulse_b200.ztask_reset import ZTaskResetB200
    n = 2051
    raw, ids = _bad_list(n)
    tag = f"{kind} bad ids"
    if kind == "smplx":
        d = _state(n, _lib.SMPLX_BODIES, _lib.SMPLX_DOF, seed=3)
        d0 = {k: v.clone() for k, v in d.items()}
        ws, check = _smplx_run(rep, tag, smplx, d, raw, False)
    elif kind == "terrain":
        d = _state(n, 24, 69, seed=3)
        d0 = {k: v.clone() for k, v in d.items()}
        ws, check = _terrain_run(rep, tag, smpl, terrain, d, raw, True, False)
    else:
        t, ml, floor = smpl
        d = _state(n, 24, 69, seed=3, width=195)
        d0 = {k: v.clone() for k, v in d.items()}
        ws = _ztask_run(ZTaskResetB200(kind, ml, floor), d, kind, 24, 69, raw, None, True)
        torch.cuda.synchronize()
        check = lambda i: _check_ztask(rep, tag, t, ml, floor, kind, True, d, i.to(DEV), 24, 69, True, 195)
    assert int(ws["count"].item()) == ids.numel() and torch.equal(ws["env_list"][:ids.numel()].cpu(), ids)
    check(ids)
    _untouched(d, d0, ids, n)


# ---------------------------------------------------------------------------------------------------------------- reference state, getup
def _im_state(n, seed, P=0):
    g = torch.Generator().manual_seed(seed)
    d = {"motion_ids": torch.randint(0, CLIPS, (n,), generator=g), "start_times": torch.rand(n, generator=g),
         "start_offset": torch.rand(n, generator=g), "global_offset": torch.randn(n, 3, generator=g),
         "progress_buf": torch.randint(0, 300, (n,), generator=g), "reset_buf": torch.zeros(n, dtype=torch.int64),
         "terminate_buf": (torch.rand(n, generator=g) < 0.5).long(), "cycle_counter": torch.randint(0, 9, (n,), generator=g, dtype=torch.int32),
         "root_all": torch.randn(n, 2, 13, generator=g), "dof_state": torch.randn(n, 72, 2, generator=g), "body": torch.randn(n, 26, 13, generator=g),
         "contact": torch.randn(n, 26, 3, generator=g), "amp": torch.randn(n, STEPS, 196, generator=g)}
    if P:
        d.update(recovery_counter=torch.randint(0, 9, (n,), generator=g, dtype=torch.int32), avail=(torch.rand(P, generator=g) < 0.4).long(),
                 fid=torch.randint(0, P, (n,), generator=g), fall_root=torch.randn(P, 13, generator=g), fall_dof=torch.randn(P, 69, 2, generator=g))
    return {k: v.to(DEV) for k, v in d.items()}


IM_KEYS = ("motion_ids", "start_times", "start_offset", "global_offset", "progress_buf", "reset_buf", "terminate_buf", "cycle_counter",
           "root_all", "dof_state", "body", "contact", "amp")


def _im_kw(d):
    return dict(motion_ids=d["motion_ids"], motion_start_times=d["start_times"], motion_start_offset=d["start_offset"],
                global_offset=d["global_offset"], progress_buf=d["progress_buf"], root_states=d["root_all"][:, 0], dof_pos=d["dof_state"][:, :69, 0],
                dof_vel=d["dof_state"][:, :69, 1], rigid_body_state=d["body"], terminate_buf=d["terminate_buf"], cycle_counter=d["cycle_counter"],
                contact_forces=d["contact"], amp_obs_buf=d["amp"], seed=SEED, offset=OFF)


def _check_ref_state(rep, tag, t, d, ids):
    """The reference-state envs: start time from word x, the motion as gathered (no ground fix, no adjustment), every AMP row from the
    motion at t0 - k dt (dt = the step's 1/30 s)."""
    idd = ids.to(DEV)
    mids = d["motion_ids"][idd].cpu()
    ph = rf.uniform(rf.words(SEED, ids.numpy().astype(np.uint64), OFF)[:, 0])
    t0 = rf.start_time_ref(ph, t["lengths"][mids])
    rf.check_exact(rep, f"{tag} start time", d["start_times"][idd].cpu(), t0)
    td = {k: v.to(DEV) for k, v in t.items()}
    ref = rf.reset_state_ref(td, mids.to(DEV), t0.to(DEV), None, rf.POSE_AS_IS, True)
    got = {"body": d["body"][idd, :24], "root": d["root_all"][idd, 0], "dof_pos": d["dof_state"][idd, :69, 0], "dof_vel": d["dof_state"][idd, :69, 1]}
    rf.check_state(rep, tag, got, ref)
    rf.check_exact(rep, f"{tag} counters", torch.stack([d["progress_buf"][idd], d["reset_buf"][idd], d["terminate_buf"][idd],
                                                        d["cycle_counter"][idd].long()]).cpu(), torch.zeros(4, len(ids), dtype=torch.int64))
    times = rf.history_times(t0, float(np.float32(1.0 / 30.0)), STEPS)
    for k in range(STEPS):
        rf.check_amp(rep, f"{tag} row {k}", d["amp"][idd, k], rf.motion_amp_ref(rf.motion_ref(td, mids.to(DEV), times[:, k].to(DEV)), True))


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("frac", [0.05, 1.0])
def test_ref_state_reset(rep, smpl, n, frac):
    from pulse_b200.humanoid_im import HumanoidImCompute
    t, ml, _ = smpl
    comp = HumanoidImCompute(ml)
    ids = _ids(n, frac, n + 4)
    runs = []
    for inject in (True, False):
        d = _im_state(n, seed=n)
        d0 = {k: v.clone() for k, v in d.items()}
        kw = _im_kw(d)
        if _mode(n, frac) == "mask":
            d["reset_buf"][ids.to(DEV)] = 1
            kw["reset_buf"] = d["reset_buf"]
        else:
            kw["env_ids"] = ids.to(DEV)
        if inject:
            kw["phase"] = rf.uniform(rf.words(SEED, np.arange(n, dtype=np.uint64), OFF)[:, 0]).to(DEV)
        ws = comp.reset_envs(**kw)
        torch.cuda.synchronize()
        assert int(ws["count"].item()) == ids.numel() and torch.equal(ws["env_list"][:ids.numel()].cpu(), ids)
        _check_ref_state(rep, f"ref state n={n} {frac}{' injected' if inject else ''}", t, d, ids)
        _untouched(d, d0, ids, n, IM_KEYS)
        runs.append(d)
    _same(runs[0], runs[1], f"ref state n={n}")


@pytest.mark.parametrize("n,P", [(1, 4), (257, 64), (2051, 300), (16384, 2000)])
@pytest.mark.parametrize("frac", [0.05, 1.0])
def test_getup_reset(rep, smpl, n, P, frac):
    from pulse_b200.humanoid_im import HumanoidImCompute
    t, ml, _ = smpl
    ids = _ids(n, frac, n + 5)
    p_rec, p_fall, steps = 0.4, 0.7, 60
    runs = []
    for inject in (True, False):
        comp = HumanoidImCompute(ml)
        d = _im_state(n, seed=n + 7, P=P)
        d0 = {k: v.clone() for k, v in d.items()}
        kw = _im_kw(d)
        if _mode(n, frac) == "mask":
            d["reset_buf"][ids.to(DEV)] = 1
            kw["reset_buf"] = d["reset_buf"]
        else:
            kw["env_ids"] = ids.to(DEV)
        if inject:
            full = rf.getup_draws(SEED, np.arange(n), OFF, P)
            kw.update(phase=full["phase"].to(DEV), recovery_u=full["recovery_u"].to(DEV), fall_u=full["fall_u"].to(DEV),
                      fall_keys=rf.bits_as_float(full["key_bits"]).to(DEV))
        ws = comp.reset_getup(**kw, recovery_counter=d["recovery_counter"], available_fall_states=d["avail"], fall_id_assignments=d["fid"],
                              fall_root_states=d["fall_root"], fall_dof_pos=d["fall_dof"][..., 0], fall_dof_vel=d["fall_dof"][..., 1],
                              recovery_prob=p_rec, fall_prob=p_fall, recovery_steps=steps)
        torch.cuda.synchronize()
        tag = f"getup n={n} P={P} {frac}{' injected' if inject else ''}"
        dr = rf.getup_draws(SEED, np.arange(n), OFF, P)
        want = rf.getup_ref(ids, d0["terminate_buf"].cpu(), d0["avail"].cpu(), d0["fid"].cpu(), dr["recovery_u"], dr["fall_u"], dr["key_bits"],
                            p_rec, p_fall, steps, d0["recovery_counter"].cpu())
        cc = ws["class_counts"].cpu()
        rf.check_exact(rep, f"{tag} class counts", cc, want["class_counts"])
        rf.check_exact(rep, f"{tag} union list", ws["env_list"][:int(ws["count"].item())].cpu(), ids)
        for k, c in (("ref_list", 0), ("fall_list", 1), ("recovery_list", 2)):
            rf.check_exact(rep, f"{tag} {k}", ws[k][:int(cc[c])].cpu(), want[k])
        rf.check_exact(rep, f"{tag} fall_pick", ws["fall_pick"][:int(cc[1])].cpu(), want["fall_pick"])
        rf.check_exact(rep, f"{tag} error", ws["error"].cpu(), torch.tensor([want["error"]]))
        rf.check_exact(rep, f"{tag} env class", ws["env_class"][ids.to(DEV)].cpu().long(), want["env_class"].long())
        for k, w in (("recovery_counter", "counter"), ("avail", "avail"), ("fid", "assign")):
            rf.check_exact(rep, f"{tag} {k}", d[k].cpu(), want[w])
        fl, pk = want["fall_list"].to(DEV), want["fall_pick"].to(DEV)
        rf.check_exact(rep, f"{tag} fall root copy", d["root_all"][fl, 0].cpu(), d0["fall_root"][pk].cpu())
        rf.check_exact(rep, f"{tag} fall dof copy", d["dof_state"][fl, :69].cpu(), d0["fall_dof"][pk].cpu())
        if want["ref_list"].numel():
            _check_ref_state(rep, tag + " ref", t, d, want["ref_list"])
        # getup_amp_init after the refresh: row 0 of the fall and recovery envs from their state, repeated into every row of a fall env
        comp.getup_amp_init(body_state=d["body"], dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1], amp_obs_buf=d["amp"])
        torch.cuda.synchronize()
        both = torch.cat([want["fall_list"], want["recovery_list"]]).to(DEV)
        if both.numel():
            rf.check_amp(rep, f"{tag} amp init row 0", d["amp"][both, 0],
                         rf.state_amp_ref(d["body"][both], d["dof_state"][both, :69, 0], d["dof_state"][both, :69, 1], True))
        if fl.numel():
            rf.check_exact(rep, f"{tag} amp init repeats row 0", d["amp"][fl].cpu(), d["amp"][fl, :1].expand(-1, STEPS, -1).cpu())
        rec = want["recovery_list"].to(DEV)
        if rec.numel():
            rf.check_exact(rep, f"{tag} amp init recovery rows k > 0", d["amp"][rec, 1:].cpu(), d0["amp"][rec, 1:].cpu())
        _untouched(d, d0, ids, n, IM_KEYS)
        runs.append(d)
    _same(runs[0], runs[1], f"getup n={n}")
