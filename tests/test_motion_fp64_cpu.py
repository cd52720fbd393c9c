"""The motion library's float64 references (tests/motion_fp64.py) have teeth: an fp32 CPU simulation of each kernel passes its link, and a
simulation with one defect fails it with BoundError naming that link.  The simulations restate the kernels' arithmetic (motion_loader.cu,
motionlib.cu, quat_math.cuh) in float32 torch operations, with float64 where the kernels use it."""
import math

import pytest
import torch

from oracle import pulse_oracle as po
from tests import motion_fp64 as mf
from tests.helpers import exact_tables

F32 = torch.float32
RATES = [24.0, 25.0, 29.97, 30.0, 50.0, 60.0, 120.0, 30.0, 60.0]
LENGTHS = [2, 3, 8, 9, 16, 17, 18, 40, 1]


# ---------------------------------------------------------------------------------------------------------------- fp32 simulations
def qmul8_32(a, b):
    """quat_math.cuh qmul in float32."""
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    ww = (az + ax) * (bx + by)
    yy = (aw - ay) * (bw + bz)
    zz = (aw + ay) * (bw - bz)
    xx = ww + yy + zz
    qq = 0.5 * (xx + (az - ax) * (bx - by))
    return torch.stack([qq - xx + (ax + aw) * (bx + bw), qq - yy + (aw - ax) * (by + bz), qq - zz + (az + ay) * (bw - bx),
                        qq - ww + (az - ay) * (by - bz)], -1)


def slerp32(a, b, t, flip=True):
    c = (a * b).sum(-1, keepdim=True)
    if flip:
        b = torch.where(c < 0, -b, b)
    c = c.abs() if flip else c
    s = torch.sqrt(torch.clamp(1.0 - c * c, min=0.0))
    h = torch.acos(torch.clamp(c, -1.0, 1.0))
    y = torch.sin((1.0 - t) * h) / s * a + torch.sin(t * h) / s * b
    y = torch.where(s.abs() < 0.001, 0.5 * a + 0.5 * b, y)
    return torch.where(c >= 1.0, a, y)


def expmap32(q, wrap=True):
    w = q[..., 3:]
    s = torch.sqrt(1.0 - w * w)
    ang = 2.0 * torch.acos(w)
    if wrap:
        ang = torch.where(ang >= mf.PI32, ang - mf.TWO_PI32, ang)
    e = ang / s * q[..., :3]
    return torch.where(s.abs() > 1e-5, e, torch.zeros_like(e))


def fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def sim_pose(quat, trans, frame_clip, headings, parents, loc, mut=None):
    g = quat.clone()
    hsign = -1.0 if mut == "heading_transposed" else 1.0
    if headings is not None:
        h = headings[frame_clip.long()]
        r = torch.stack([torch.zeros_like(h), torch.zeros_like(h), hsign * torch.sin(0.5 * h), torch.cos(0.5 * h)], -1)[:, None]
        g = mf.qmul(r.expand_as(g), g / g.norm(dim=-1, keepdim=True))
    lr = torch.stack([g[:, j] if p < 0 else mf.qnormalize(mf.qmul(mf.qconj(g[:, p]), g[:, j])) for j, p in enumerate(parents)], 1)
    lf = lr.float()
    t = trans.clone()
    if headings is not None:
        c, s = torch.cos(h), torch.sin(h)
        t = torch.stack([c * t[:, 0] - s * t[:, 1], s * t[:, 0] + c * t[:, 1], t[:, 2]], -1)
    rot, pos = [None] * 24, [None] * 24
    for j, p in enumerate(parents):
        if p < 0:
            rot[j], pos[j] = lf[:, j], t.float()
        else:
            rot[j] = mf.qnormalize(mf.qmul(rot[p], lf[:, j]))
            pos[j] = mf.qrotate(rot[p], loc[j].expand(len(t), 3)) + pos[p]
    return g.float(), lf, torch.stack(pos, 1)


def sim_velocity(gts, lrs, quat, frame_clip, clip_start, fps, headings, mut=None):
    F = gts.shape[0]
    f = torch.arange(F)
    f0, f1 = mf.clip_bounds(frame_clip, clip_start)
    fps32 = fps.float()
    if mut == "dt_30":
        fps32 = torch.full_like(fps32, 30.0)
    dt = 1.0 / fps32.double()[frame_clip.long()]
    if mut == "central_at_ends":
        fa, fb = (f - 1).clamp(0, F - 1), (f + 1).clamp(0, F - 1)
    else:
        fa, fb = torch.where(f > f0, f - 1, f), torch.where(f + 1 < f1, f + 1, f)
    inv = 1.0 / ((fb - fa).double() * dt).float()
    vel = torch.where((fb > fa)[:, None, None], (gts[fb] - gts[fa]) * inv[:, None, None], torch.zeros_like(gts))
    g = quat.double()
    if headings is not None:
        h = headings[frame_clip.long()]
        r = torch.stack([torch.zeros_like(h), torch.zeros_like(h), torch.sin(0.5 * h), torch.cos(0.5 * h)], -1)[:, None]
        g = mf.qmul(r.expand_as(g), g / g.norm(dim=-1, keepdim=True))
    has_next = f + 1 < f1
    nxt = torch.where(has_next, f + 1, f)
    if mut == "last_ang_nonzero":
        nxt = torch.where(has_next, f + 1, (f - 1).clamp(min=0))
        has_next = f >= 0
    d = mf.qnormalize(mf.qmul(g[nxt], mf.qconj(g)))
    ang = torch.acos(torch.clamp(2 * d[..., 3] ** 2 - 1, -1, 1))
    n = d[..., :3].norm(dim=-1).clamp_min(1e-9)
    w = d[..., :3] * (ang / (n * dt[:, None]))[..., None]
    if mut == "last_ang_nonzero":
        last = f + 1 == f1
        w[last] = -w[last]
    w = torch.where(has_next[:, None, None], w, torch.zeros_like(w)).float()
    fs = torch.where(f + 1 < f1, f, f - 1)
    if mut == "dof_pair_back":
        fs = torch.where(f > f0, f - 1, f)
    pair = (fs >= f0) & (fs + 1 < f1)
    fs_c, fs1 = torch.where(pair, fs, f), torch.where(pair, fs + 1, f)
    e = expmap32(qmul8_32(mf.qconj(lrs[fs_c, 1:]), lrs[fs1, 1:]))
    r = (1.0 / dt).float()
    dv = torch.where(pair[:, None, None], e * r[:, None, None], torch.zeros_like(e))
    return vel, w, dv


def sim_filter(tmp_vel, tmp_ang, frame_clip, clip_start, mut=None):
    F = tmp_vel.shape[0]
    k = torch.arange(-8, 9)
    w = torch.exp(-0.5 * (k * k).float() / 4.0)
    wsum = w[8].clone()
    for i in range(1, 9):
        wsum = wsum + 2.0 * w[8 + i]
    wk = w / wsum
    f = torch.arange(F)
    t = f[:, None] + k[None, :]
    if mut == "global_clamp":
        taps = t.clamp(0, F - 1)
    elif mut == "reflect":
        f0, f1 = mf.clip_bounds(frame_clip, clip_start)
        lo, hi = f0[:, None], f1[:, None] - 1
        taps = torch.where(t < lo, 2 * lo - t - 1, torch.where(t > hi, 2 * hi - t + 1, t))
        taps = torch.minimum(torch.maximum(taps, lo), hi)
    else:
        taps = mf.filter_taps(frame_clip, clip_start)
    outs = []
    for x in (tmp_vel, tmp_ang):
        acc = torch.zeros_like(x)
        for i in range(17):
            acc = fma32(wk[i].expand_as(x), x[taps[:, i]], acc)
        outs.append(acc)
    return outs


def sim_query(tb, ids, times, offset=None, mut=None, bodies=24):
    i0, i1, b = po.frame_blend(times, tb["lengths"][ids], tb["num_frames"][ids], tb["dt"][ids])
    if mut == "unclamped_blend":
        b = (torch.where(times < 0, torch.zeros_like(times), times) - i0 * tb["dt"][ids]) / tb["dt"][ids]
    f0, f1 = i0 + tb["length_starts"][ids], i1 + tb["length_starts"][ids]
    bb = b[:, None, None]
    lerp = lambda k: (1.0 - bb) * tb[k][f0] + bb * tb[k][f1]
    pos = lerp("gts")
    if offset is not None:
        pos = pos + offset[:, None, :]
    rot = slerp32(tb["grs"][f0], tb["grs"][f1], bb, flip=mut != "no_sign_flip")
    loc = slerp32(tb["lrs"][f0][:, 1:], tb["lrs"][f1][:, 1:], bb, flip=mut != "no_sign_flip")
    dof = expmap32(loc, wrap=mut != "no_wrap")
    out = {"frame_idx0": i0, "frame_idx1": i1, "blend": b, "rg_pos": pos, "rb_rot": rot, "body_vel": lerp("gvs"), "body_ang_vel": lerp("gavs"),
           "dof_vel": lerp("dvs").reshape(len(ids), -1), "dof_pos": dof.reshape(len(ids), -1)}
    if "motion_aa" in tb:
        out["motion_aa"] = tb["motion_aa"][f0]
    if mut == "smplx_slot":                                # lane l writes body l + 32 into slot l + 31
        for k in ("rg_pos", "rb_rot", "body_vel", "body_ang_vel"):
            v = out[k].clone()
            v[:, 31:bodies - 1] = out[k][:, 32:]
            out[k] = v
    out.update(root_pos=out["rg_pos"][:, 0], root_rot=out["rb_rot"][:, 0], root_vel=out["body_vel"][:, 0], root_ang_vel=out["body_ang_vel"][:, 0])
    return out


# ---------------------------------------------------------------------------------------------------------------- inputs
def _loader_inputs(headings="mixed"):
    return mf.loader_clips(LENGTHS, RATES, seed=11, headings=headings)


def _check_loader(mut=None, headings="mixed"):
    quat, trans, fc, cs, fps, hd, loc = _loader_inputs(headings)
    grs, lrs, gts = sim_pose(quat, trans, fc, hd, mf.SMPL_PARENTS, loc, mut)
    ref = mf.loader_pose_ref(quat, trans, fc, hd, mf.SMPL_PARENTS, loc, lrs)
    mf.check(None, "pose grs", grs, *ref["grs"])
    lr, lt, amb = ref["lrs"]
    mf.check_branches(None, "pose lrs", lrs, [(lr, lt, torch.ones(amb.shape, dtype=torch.bool)), (-lr, lt, amb)])
    mf.check(None, "pose gts", gts, *ref["gts"])
    tv, ta, dv = sim_velocity(gts, lrs, quat, fc, cs, fps, hd, mut)
    vr = mf.loader_velocity_ref(gts, lrs, quat, fc, cs, fps, hd)
    mf.check(None, "velocity tmp_vel", tv, *vr["tmp_vel"])
    mf.check(None, "velocity tmp_ang", ta, *vr["tmp_ang"])
    mf.check_branches(None, "velocity dvs", dv, vr["dvs"])
    gv, ga = sim_filter(tv, ta, fc, cs, mut)
    fr = mf.loader_filter_ref(tv, ta, fc, cs)
    mf.check(None, "filter gvs", gv, *fr["gvs"])
    mf.check(None, "filter gavs", ga, *fr["gavs"])


def _query_tables(smplx=False):
    """exact_tables at mixed rates (SMPL) or 52-body tables (SMPL-X), with built rows: clip 3 frames 0/1 antipodal, 1/2 identical, 2/3
    nearly identical (s ~ 1e-4, the midpoint), 3/4 local rotations with w = +-1e-3 (near pi)."""
    if smplx:
        from tests.smplx_speed_oracle import tables
        tb = tables(12, seed=4)
        rates = mf_rates(12)
        nf = tb.num_frames
        tb.dt = (1.0 / rates).float()
        tb.lengths = ((nf - 1).double() * (1.0 / rates)).float()
    else:
        tb = exact_tables(12, seed=4, fps=RATES[:7])
    t = {k: getattr(tb, k).clone() if torch.is_tensor(getattr(tb, k)) else getattr(tb, k) for k in
         ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames", "dt", "length_starts")}
    build_branch_rows(t, clip=3)
    return t


def mf_rates(m):
    from tests.helpers import clip_rates
    return clip_rates(RATES[:7], m)


def build_branch_rows(t, clip):
    """Frames 0..4 of `clip` put each slerp / exp-map branch on every body (bodies >= 32 included for SMPL-X)."""
    s = int(t["length_starts"][clip])
    assert int(t["num_frames"][clip]) >= 6
    for k in ("grs", "lrs"):
        q = t[k]
        q[s + 1] = -q[s]                                          # antipodal: c = -1 (the sign flip, then c >= 1)
        q[s + 2] = q[s + 1]                                       # identical: c >= 1
        q[s + 3] = torch.nn.functional.normalize(q[s + 2] + 1e-4 * q[s + 2].roll(1, -1), dim=-1)   # nearly identical: s ~ 1e-4
    near_pi = torch.nn.functional.normalize(torch.randn(t["lrs"].shape[1], 3, generator=torch.Generator().manual_seed(1)), dim=-1)
    t["lrs"][s + 4, :, :3] = near_pi * math.sqrt(1 - 1e-6)
    t["lrs"][s + 4, :, 3] = torch.where(torch.arange(t["lrs"].shape[1]) % 2 == 0, 1e-3, -1e-3)
    t["lrs"][s + 5] = t["lrs"][s + 4]


def query_times(t, ids):
    """Per query: negative, zero, on-frame multiples, the length, past it, random."""
    g = torch.Generator().manual_seed(8)
    n = ids.shape[0]
    L, dt, nf = t["lengths"][ids], t["dt"][ids], t["num_frames"][ids]
    k = torch.randint(0, 1 << 20, (n,), generator=g) % nf
    kinds = torch.arange(n) % 6
    times = torch.rand(n, generator=g) * L
    times = torch.where(kinds == 0, -torch.rand(n, generator=g), times)
    times = torch.where(kinds == 1, torch.zeros_like(times), times)
    times = torch.where(kinds == 2, k.float() * dt, times)
    times = torch.where(kinds == 3, L, times)
    times = torch.where(kinds == 4, L + torch.rand(n, generator=g), times)
    return times


def branch_queries(t, clip):
    """Queries at the built frames: between each built pair at blends 0.25 / 0.5 / 0.75."""
    s = t["dt"][clip]
    ids = torch.full((15,), clip, dtype=torch.int64)
    fr = torch.arange(5).repeat_interleave(3).float()
    bl = torch.tensor([0.25, 0.5, 0.75]).repeat(5)
    return ids, ((fr + bl) * s.double()).float()


def _check_query(mut=None, smplx=False, offset=True):
    t = _query_tables(smplx)
    n = 600
    ids = torch.arange(n) % t["lengths"].shape[0]
    times = query_times(t, ids)
    bid, btimes = branch_queries(t, 3)
    ids, times = torch.cat([ids, bid]), torch.cat([times, btimes])
    built = torch.zeros(ids.shape[0], dtype=torch.bool)
    built[n:] = True
    off = torch.randn(ids.shape[0], 3, generator=torch.Generator().manual_seed(2)) if offset else None
    B = t["gts"].shape[1]
    got = sim_query(t, ids, times, off, mut, bodies=B)
    if smplx:
        got.pop("motion_aa", None)
    ref = mf.query_ref(t if not smplx else {k: v for k, v in t.items() if k != "motion_aa"}, ids, times, got["blend"], off)
    mf.check_query(None, "query", got, ref, built=built)


# ---------------------------------------------------------------------------------------------------------------- tests
def test_simulated_loader_passes_every_link():
    _check_loader()
    _check_loader(headings=None)


@pytest.mark.parametrize("mut,link", [("global_clamp", "filter gvs"), ("reflect", "filter gvs"), ("central_at_ends", "velocity tmp_vel"),
                                      ("dt_30", "velocity tmp_vel"), ("heading_transposed", "pose grs"), ("dof_pair_back", "velocity dvs"),
                                      ("last_ang_nonzero", "velocity tmp_ang")])
def test_loader_mutation_fails_its_link(mut, link):
    with pytest.raises(mf.BoundError, match=link):
        _check_loader(mut)


@pytest.mark.parametrize("smplx", [False, True])
def test_simulated_query_passes_every_link(smplx):
    _check_query(smplx=smplx)
    _check_query(smplx=smplx, offset=False)


@pytest.mark.parametrize("mut,link,smplx", [("no_sign_flip", "rb_rot", False), ("unclamped_blend", "blend", False),
                                            ("no_wrap", "dof_pos", False), ("smplx_slot", "rg_pos", True), ("no_sign_flip", "rb_rot", True),
                                            ("no_wrap", "dof_pos", True)])
def test_query_mutation_fails_its_link(mut, link, smplx):
    with pytest.raises(mf.BoundError, match=link):
        _check_query(mut, smplx=smplx)


def test_fma_in_the_motion_time_flips_a_frame_index_on_frame():
    """The step's motion time progress * dt + start (two fp32 roundings, motion_time_rn) with a fused multiply-add instead: at start times on
    the 1/30 s grid the product lands on frame boundaries, and one rounding fewer moves some of them across."""
    t = exact_tables(40, seed=4, fps=RATES[:7])
    M = 40
    prog = torch.arange(0, 60).repeat(M)
    ids = torch.arange(M).repeat_interleave(60)
    start = (torch.arange(M * 60) % 7).double().mul(1.0 / 30).float()
    dt = po.STEP_DT
    ref_t = po.im_motion_times(prog, start, torch.zeros_like(start), dt, plus_one=False)
    fma_t = fma32(prog.float(), torch.full_like(start, dt), start)
    i0r, _, _ = po.frame_blend(ref_t, t.lengths[ids], t.num_frames[ids], t.dt[ids])
    i0m, _, _ = po.frame_blend(fma_t, t.lengths[ids], t.num_frames[ids], t.dt[ids])
    mf.check_exact(None, "frame_idx0 (motion time)", i0r, po.frame_blend(ref_t, t.lengths[ids], t.num_frames[ids], t.dt[ids])[0])
    with pytest.raises(mf.BoundError, match="frame_idx0"):
        mf.check_exact(None, "frame_idx0 (motion time)", i0m, i0r)


def test_packed_records_layout():
    t = exact_tables(5, seed=1, fps=RATES[:5])
    d = {k: getattr(t, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa")}
    fr, ax = mf.packed_records(d)
    assert fr.shape[1] == mf.FRAME_REC and ax.shape[1] == mf.AUX_REC
    assert torch.equal(fr[:, 72:168], t.grs.reshape(-1, 96)) and torch.equal(ax[:, 165:237], t.motion_aa) and not ax[:, 237:].any()


def test_slerp_weight_slope_bound():
    """|d/dh sin((1 - t) h) / sin h| <= 0.25 h over (0, pi/2] and t in [0, 1] (slerp_cands relies on it)."""
    h = torch.linspace(1e-4, math.pi / 2, 2000, dtype=torch.float64)[:, None]
    t = torch.linspace(0, 1, 201, dtype=torch.float64)[None, :]
    R = lambda x: torch.sin((1 - t) * x) / torch.sin(x)
    d = (R(h + 1e-7) - R(h - 1e-7)) / 2e-7
    assert float((d.abs() / h).max()) <= 0.25
