"""The motion library's kernels element-wise against the float64 references of tests/motion_fp64.py, at clip rates 24 to 120 fps: the
device loader's three passes (teacher-forced through their own workspaces), the record packing, and the SMPL and SMPL-X queries at times
before, on, between and past the frames, with rows built on every branch of slerp and of the exponential map.  `-s` prints every margin."""
import ctypes as C

import pytest
import torch

from tests import motion_fp64 as mf
from tests.helpers import clip_rates, exact_tables
from tests.test_motion_fp64_cpu import build_branch_rows, branch_queries, query_times

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
RATES = [24.0, 25.0, 29.97, 30.0, 50.0, 60.0, 120.0]
KEYS = ("gts", "grs", "lrs", "gvs", "gavs", "dvs")


@pytest.fixture(scope="module")
def rep():
    r = mf.Report("motion library vs float64 references")
    yield r
    print("\n" + r.text())


def _load(quat, trans, fc, cs, fps, hd, loc):
    """pulse_motionlib_load_clips with the test's own workspaces: the six tables and tmp_vel / tmp_ang."""
    from pulse_b200 import _lib
    lib = _lib.load()
    F = quat.shape[0]
    z = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.float32)
    t = {"gts": z(F, 24, 3), "grs": z(F, 24, 4), "lrs": z(F, 24, 4), "gvs": z(F, 24, 3), "gavs": z(F, 24, 3), "dvs": z(F, 23, 3),
         "tmp_vel": z(F, 24, 3), "tmp_ang": z(F, 24, 3)}
    ins = dict(quat=quat.to(DEV, torch.float64).contiguous(), trans=trans.to(DEV, torch.float64).contiguous(), fc=fc.to(DEV, torch.int32).contiguous(),
               cs=cs.to(DEV, torch.int64).contiguous(), fps=fps.to(DEV, torch.float32).contiguous(),
               hd=None if hd is None else hd.to(DEV, torch.float64).contiguous(), par=torch.tensor(mf.SMPL_PARENTS, dtype=torch.int32, device=DEV),
               loc=loc.to(DEV, torch.float32).contiguous())
    a = _lib.LoaderArgs(pose_quat_global=ins["quat"].data_ptr(), root_trans=ins["trans"].data_ptr(), frame_clip=ins["fc"].data_ptr(),
                        clip_start=ins["cs"].data_ptr(), fps=ins["fps"].data_ptr(), headings=_lib.ptr(ins["hd"]), parents=ins["par"].data_ptr(),
                        local_translation=ins["loc"].data_ptr(), total_frames=F, num_clips=len(fps),
                        **{k: t[k].data_ptr() for k in t})
    _lib.check(lib.pulse_motionlib_load_clips(C.byref(a), _lib.current_stream(DEV)), "pulse_motionlib_load_clips")
    torch.cuda.synchronize()
    return t


def _check_loader(rep, tag, inputs):
    quat, trans, fc, cs, fps, hd, loc = inputs
    k = _load(*inputs)
    d = lambda x: None if x is None else x.to(DEV)
    quat, trans, fc, cs, fps64, hd, loc = d(quat), d(trans), d(fc), d(cs), d(fps), d(hd), d(loc)
    ref = mf.loader_pose_ref(quat, trans, fc, hd, mf.SMPL_PARENTS, loc, k["lrs"])
    mf.check(rep, f"{tag} pose grs", k["grs"], *ref["grs"])
    lr, lt, amb = ref["lrs"]
    mf.check_branches(rep, f"{tag} pose lrs", k["lrs"], [(lr, lt, torch.ones_like(amb)), (-lr, lt, amb)])
    mf.check(rep, f"{tag} pose gts (FK)", k["gts"], *ref["gts"])
    vr = mf.loader_velocity_ref(k["gts"], k["lrs"], quat, fc, cs, fps64, hd)
    mf.check(rep, f"{tag} velocity tmp_vel", k["tmp_vel"], *vr["tmp_vel"])
    mf.check(rep, f"{tag} velocity tmp_ang", k["tmp_ang"], *vr["tmp_ang"])
    mf.check_branches(rep, f"{tag} velocity dvs", k["dvs"], vr["dvs"])
    fr = mf.loader_filter_ref(k["tmp_vel"], k["tmp_ang"], fc, cs)
    mf.check(rep, f"{tag} filter gvs", k["gvs"], *fr["gvs"])
    mf.check(rep, f"{tag} filter gavs", k["gavs"], *fr["gavs"])
    return k


def _loader_set(headings="mixed"):
    lengths = [2, 3, 8, 9, 16, 17, 18, 1000, 1213, 2, 17, 9, 40, 5]
    return mf.loader_clips(lengths, [RATES[i % 7] for i in range(len(lengths))], seed=21, headings=headings)


def _tables_from_loader(k, inputs):
    fps = inputs[4]
    nf = (inputs[3][1:] - inputs[3][:-1]).to(torch.int64)
    t = {key: k[key].cpu() for key in KEYS}
    t.update(lengths=torch.tensor([1.0 / r * (int(n) - 1) for r, n in zip(fps.tolist(), nf)], dtype=torch.float32), num_frames=nf,
             dt=(1.0 / fps).float(), length_starts=inputs[3][:-1].clone(), motion_aa=torch.zeros(k["gts"].shape[0], 72))
    return t


def test_loader_mixed_rates(rep):
    _check_loader(rep, "loader mixed", _loader_set())
    _check_loader(rep, "loader no heading", _loader_set(headings=None))


def test_loader_at_scale(rep):
    g = torch.Generator().manual_seed(5)
    lengths = (torch.randint(1, 48, (3000,), generator=g)).tolist()
    inputs = mf.loader_clips(lengths, [RATES[i % 7] for i in range(len(lengths))], seed=22)
    _check_loader(rep, "loader 3000 clips", inputs)


def _mlib(t):
    from pulse_b200.motion_lib import MotionLibB200
    return MotionLibB200.from_tables({k: v for k, v in t.items()}, device=DEV)


def _smpl_tables():
    tb = exact_tables(40, seed=4, fps=RATES)
    t = {k: getattr(tb, k).clone() for k in KEYS + ("motion_aa", "lengths", "num_frames", "dt", "length_starts")}
    build_branch_rows(t, clip=3)
    return t


def _smplx_tables():
    from tests.smplx_speed_oracle import tables
    tb = tables(40, seed=4)
    rates = clip_rates(RATES, 40)
    t = {k: getattr(tb, k).clone() for k in KEYS + ("num_frames", "length_starts")}
    t.update(dt=(1.0 / rates).float(), lengths=((tb.num_frames - 1).double() * (1.0 / rates)).float())
    build_branch_rows(t, clip=3)
    return t


def test_packing_bit_exact(rep):
    t = _smpl_tables()
    ml = _mlib(t)
    fr, ax = mf.packed_records(t)
    mf.check_exact(rep, "pack frame_rec", ml.frame_rec.cpu(), fr)
    mf.check_exact(rep, "pack aux_rec", ml.aux_rec.cpu(), ax)
    tx = _smplx_tables()
    mx = _mlib(tx)
    fr, ax = mf.packed_records(tx, smplx=True)
    mf.check_exact(rep, "pack smplx frame_rec", mx.frame_rec.cpu(), fr)
    mf.check_exact(rep, "pack smplx aux_rec", mx.aux_rec.cpu(), ax)


def _queries(t, n, seed):
    M = t["lengths"].shape[0]
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, M, (n,), generator=g)
    times = query_times(t, ids)
    built = torch.zeros(n, dtype=torch.bool)
    if n >= 15:
        bid, bt = branch_queries(t, 3)
        ids[:15], times[:15], built[:15] = bid, bt, True
    return ids, times, built


def _run_query(rep, tag, t, n, offset, smplx):
    ml = _mlib(t)
    ids, times, built = _queries(t, n, seed=n)
    off = torch.randn(n, 3, generator=torch.Generator().manual_seed(3)) if offset else None
    out = ml.get_motion_state(ids.to(DEV), times.to(DEV), None if off is None else off.to(DEV), diagnostics=not smplx)
    torch.cuda.synchronize()
    got = {k: v for k, v in out.items() if k not in ("motion_bodies", "motion_limb_weights")}
    if smplx:
        from oracle import pulse_oracle as po
        got["blend"] = po.frame_blend(times, t["lengths"][ids], t["num_frames"][ids], t["dt"][ids])[2].to(DEV)
    td = {k: v.to(DEV) for k, v in t.items()}
    ref = mf.query_ref(td, ids.to(DEV), times.to(DEV), got["blend"], None if off is None else off.to(DEV))
    mf.check_query(rep, tag, got, ref, built=built.to(DEV), diagnostics=not smplx)
    rp = ml.get_root_pos_smpl(ids.to(DEV), times.to(DEV))
    torch.cuda.synchronize()
    mf.check_query(rep, tag + " root_pos_smpl", rp, mf.query_ref(td, ids.to(DEV), times.to(DEV), got["blend"]), diagnostics=False)


@pytest.mark.parametrize("n", [1, 1027, 16384])
def test_query_smpl(rep, n):
    t = _smpl_tables()
    _run_query(rep, f"smpl n={n} offset", t, n, True, False)
    _run_query(rep, f"smpl n={n}", t, n, False, False)


def test_query_smpl_on_loader_tables(rep):
    inputs = _loader_set()
    k = _load(*inputs)
    _run_query(rep, "smpl loader tables", _tables_from_loader(k, inputs), 4096, True, False)


@pytest.mark.parametrize("n", [1, 1027, 16384])
def test_query_smplx(rep, n):
    _run_query(rep, f"smplx n={n} offset", _smplx_tables(), n, True, True)
    _run_query(rep, f"smplx n={n}", _smplx_tables(), n, False, True)
