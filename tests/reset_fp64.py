"""Teacher-forced float64 references of the reset kernels (reset_state.cuh, reset_warps.cuh, ztask_reset.cu, terrain_reset.cu,
getup_reset.cu) and of the AMP row of humanoid_obs.cuh, each with an element-wise bound derived from the fp32 operations its kernel
performs (the style of tests/fp64_ref.py and tests/motion_fp64.py, whose comparators and query references are reused).

Links and what feeds them:
* draws: every Philox word is regenerated on the host (tests/philox_ref.py) in the layout of include/pulse_b200.h: the reference-state
  phase x of (seed, e, off); the latent-task block r0 = (seed, e, off) with x phase, y clip, z strike near, w strike distance; the strike
  block (seed, e + 2^32, off) with x bearing, y yaw; the task block (seed, e + 2^33, off) with x, y, z the task uniforms and
  steps = steps_min + (w * span) >> 32; the terrain location (r0.z * L) >> 32; the getup recovery word y, fall word z and the fall-state
  keys (seed, s, off).w; the trajectory list's blocks (seed, e + 4 * 2^32, 101 * off + k): block k < 100 gives segment k's turn, sharp
  turn, sharp-turn coin and speed change (x, y, z, w), block 100 the initial heading and speed (x, y).
* sampling, exact: the clip pick (the kernel's binary search of the inclusive CDF for u * total, clamped below total by nextafter) and
  sample_time_interval in fp32 round-to-nearest order; the frame rows and blend of every AMP history time t0 - k dt
  (oracle.pulse_oracle.frame_blend, which tests/test_gpu_motion_fp64.py pins to the kernel's frame_blend_rn).
* reset state, teacher-forced on those rows: the lerps, slerp and exponential map through motion_fp64's candidates; the ground fix from
  floor[f0] (two roundings for d, one for the subtraction); FACE_X, a rotation about z by the inverse heading of base_rot_removed(root)
  of the bodies' positions (about the root), rotations and velocities and of the root's angular velocity, not the bodies' (as
  humanoid_speed.py does); its angle error is the first-order error of the rotated x axis over that axis' length (the root rotation's bound times 4 |q|_1, plus
  the fp32 roundings) plus 16 u32 for heading_half's rsqrt / sqrt / fdiv_fast, and every rotated vector carries |v| times that error;
  ROOT_XY_ZERO (root xy exactly 0, bodies as gathered); the strike target (dist: three roundings; theta: one rounding and fp32(2 pi);
  cosf / sinf: 2 ulp); the terrain spawn (root xy the table entry exactly; body xy shifted, z not lifted; the root lifted by the mean
  center height at the new xy, whose cells are exact unless a point lies within its bound of a cell edge).
* amp_row_ref: build_amp_observations_smpl in float64 (196 floats; 195 drops the root height), with the heading bound above, the
  rotation features of quat_to_tan_norm, and the exponential map to quaternion with its |angle| <= 1e-5 identity branch as candidates.
  Row 0 is fed the state the kernel wrote, rows k > 0 the un-fixed motion at t0 - k dt (the bounds of the gather add to the row's).
* traj_ref: TrajGenerator.reset from the start xy the kernel read (the root it wrote).  The turn angles, the clipped speed recurrence,
  the heading sum (fp32 turns added in float64, rounded to fp32) and the segment lengths are fp32 / float64 arithmetic in the kernel's
  order and are modelled exactly; the waypoints are float64 sums of cos / sin of those headings.  Bound of waypoint k: over the segments
  before it, seg (4 u32, the 2-ulp sincosf) + u32 |seg cos| (the product), the start's fp32 add, and one rounding of the float64 sum.
* getup, exact: the release of the reset envs' states, the union / reference-state / fall / recovery lists and counts, the recovery
  counters, the surplus of an exhausted pool, and fall_pick = the free states sorted by (key bits, state id).

A row whose heading is ill-conditioned (the rotated x axis shorter than four times its bound) or whose root rotation may take two
slerp branches is ambiguous: any value passes, and outside the rows a test builds there the share of such rows must stay under
AMBIGUOUS_MAX.  The same holds for terrain rows with a center point within its bound of a cell edge, under EDGE_MAX.
"""
import math
from typing import Dict, List, Optional

import numpy as np
import torch

from tests import motion_fp64 as mf
from tests.fp64_ref import U32, BoundError, Report, check, check_exact, f64  # noqa: F401  (re-exported for the tests)
from tests.philox_ref import philox4x32_10, u01

AMBIGUOUS_MAX = 1e-3
# The 3 x 3 center points are multiples of the cell size around a root on a cell corner: a yaw within a few 1e-3 rad of a multiple of
# pi / 2 puts points within their bound (about the ulp of the world coordinate) of a cell edge, and the envs that draw the same frame
# share that yaw.  Such a row is still checked, against the interval of heights its reachable cells give.
EDGE_MAX = 2e-2
STRIKE_STREAM, TASK_STREAM, TRAJ_STREAM = 1 << 32, 2 << 32, 4 << 32
TRAJ_VERTS = 101
TRAJ_SEGS = TRAJ_VERTS - 1
STEP30 = float(np.float32(1.0 / 30.0))
TWO_PI32 = float(np.float32(2.0 * math.pi))
GROUND_MARGIN = 0.02
EXP_EPS32 = float(np.float32(1e-5))
KEPT_JOINTS = [0, 1, 2, 4, 5, 6, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 19, 20, 21]
KEY_BODIES = [7, 3, 22, 17]
BASE_INV = (-0.5, -0.5, -0.5, 0.5)                  # conj(0.5, 0.5, 0.5, 0.5): remove_base_rot
POSE_AS_IS, POSE_ROOT_XY_ZERO, POSE_FACE_X = "as_is", "root_xy_zero", "face_x"


# ------------------------------------------------------------------------------------------------------------------ draws
def words(seed: int, index, offset: int) -> torch.Tensor:
    """The four Philox words of the blocks (seed, index[i], offset) as int64 [n, 4] (x, y, z, w)."""
    w = philox4x32_10(seed, np.asarray(index, dtype=np.uint64), offset)
    return torch.from_numpy(np.stack([np.asarray(c, dtype=np.int64) for c in w], 1))


def uniform(word: torch.Tensor) -> torch.Tensor:
    return torch.from_numpy(u01(word.numpy().astype(np.uint64)))


def ztask_draws(seed: int, envs, off: int) -> Dict[str, torch.Tensor]:
    """The latent-task / terrain reset draws of the envs `envs` (int64): phase, clip uniform, strike uniforms [n, 4], the raw words."""
    e = np.asarray(envs, dtype=np.uint64)
    r0, r1 = words(seed, e, off), words(seed, e + np.uint64(STRIKE_STREAM), off)
    return {"phase": uniform(r0[:, 0]), "motion_u": uniform(r0[:, 1]),
            "strike_u": torch.stack([uniform(r0[:, 2]), uniform(r0[:, 3]), uniform(r1[:, 0]), uniform(r1[:, 1])], 1), "r0": r0, "r1": r1}


def task_draws(seed: int, envs, off: int, steps_min: int, steps_max: int) -> Dict[str, torch.Tensor]:
    """pulse_ztask_reset_task's draws: uniforms [n, 3] (reach; speed takes column 0) and the randint results."""
    r = words(seed, np.asarray(envs, dtype=np.uint64) + np.uint64(TASK_STREAM), off)
    span = np.uint64(steps_max - steps_min)
    steps = steps_min + ((r[:, 3].numpy().astype(np.uint64) * span) >> np.uint64(32)).astype(np.int64)
    return {"rand": torch.stack([uniform(r[:, c]) for c in range(3)], 1), "steps": torch.from_numpy(steps)}


def terrain_loc(r0: torch.Tensor, num_locations: int) -> torch.Tensor:
    """sample_valid_locations from word z: (z * L) >> 32 in 64-bit unsigned arithmetic."""
    z = r0[:, 2].numpy().astype(np.uint64)
    return torch.from_numpy(((z * np.uint64(num_locations)) >> np.uint64(32)).astype(np.int64))


def getup_draws(seed: int, envs, off: int, num_states: int) -> Dict[str, torch.Tensor]:
    """Recovery (word y) and fall (word z) uniforms of the envs, and the key bits (word w) of every fall state s = 0 .. P - 1."""
    r = words(seed, np.asarray(envs, dtype=np.uint64), off)
    k = words(seed, np.arange(num_states, dtype=np.uint64), off)
    return {"phase": uniform(r[:, 0]), "recovery_u": uniform(r[:, 1]), "fall_u": uniform(r[:, 2]), "key_bits": k[:, 3]}


def traj_draws(seed: int, envs, off: int, stream: int = TRAJ_STREAM, counter_base=None) -> torch.Tensor:
    """pulse_traj_reset_list's draws of the envs, fp32 [n, 4 S + 2] in the injected layout: [turn | sharp angle | sharp coin | speed
    change] x S, heading, initial speed.  Block k of env e is (seed, e + stream, TRAJ_VERTS * off + k)."""
    e = np.asarray(envs, dtype=np.uint64) + np.uint64(stream)
    base = TRAJ_VERTS * off if counter_base is None else counter_base
    S = TRAJ_SEGS
    out = torch.zeros(len(e), 4 * S + 2, dtype=torch.float32)
    for k in range(S + 1):
        w = words(seed, e, base + k)
        if k < S:
            for c in range(4):
                out[:, c * S + k] = uniform(w[:, c])
        else:
            out[:, 4 * S], out[:, 4 * S + 1] = uniform(w[:, 0]), uniform(w[:, 1])
    return out


def bits_as_float(bits: torch.Tensor) -> torch.Tensor:
    """fp32 tensor with the given 32-bit patterns (what the kernel reads back with __float_as_uint)."""
    return torch.from_numpy(bits.numpy().astype(np.uint32).view(np.float32).copy())


# ------------------------------------------------------------------------------------------------------------------ sampling, exact
def pick_motion_ref(cdf: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
    """pick_motion: v = fp32(u * total), v >= total -> nextafter(total, 0), then the kernel's binary search for the first cdf > v."""
    cdf, u = cdf.float().cpu(), u.float().cpu()
    m = cdf.shape[0]
    total = cdf[m - 1]
    v = u * total
    v = torch.where(v >= total, torch.nextafter(total, torch.zeros_like(total)).expand_as(v), v)
    lo = torch.zeros_like(u, dtype=torch.int64)
    hi = torch.full_like(lo, m - 1)
    while bool((lo < hi).any()):
        live = lo < hi
        mid = (lo + hi) >> 1
        go = cdf[mid] > v
        hi = torch.where(live & go, mid, hi)
        lo = torch.where(live & ~go, mid + 1, lo)
    return lo


def start_time_ref(phase: torch.Tensor, mlen: torch.Tensor) -> torch.Tensor:
    """sample_time_interval in fp32: trunc(fp32(fp32(ph * len) / fp32(1/30))) * fp32(1/30)."""
    s = torch.tensor(STEP30, dtype=torch.float32, device=phase.device)
    k = ((phase.float() * mlen.float()).double() / STEP30).float().long()    # the fp32 quotient (innocuous double rounding)
    return k.float() * s


def history_times(t0: torch.Tensor, dt: float, steps: int) -> torch.Tensor:
    """[n, steps] query times: t0 for k = 0, fp32(t0 + fp32(-dt * k)) for k > 0."""
    k = torch.arange(steps, dtype=torch.float32)
    t = t0.float()[:, None] + (-torch.tensor(dt, dtype=torch.float32)) * k[None, :]
    t[:, 0] = t0.float()
    return t


def motion_ref(tb, mids: torch.Tensor, times: torch.Tensor) -> Dict[str, object]:
    """motion_fp64.query_ref at the exact fp32 blend, plus the global frame rows f0 / f1."""
    from oracle import pulse_oracle as po
    mids = mids.long()
    i0, i1, b = po.frame_blend(times, tb["lengths"][mids], tb["num_frames"][mids], tb["dt"][mids])
    q = mf.query_ref({k: v for k, v in tb.items() if k != "motion_aa"}, mids, times, b)
    q["f0"], q["f1"] = i0 + tb["length_starts"][mids], i1 + tb["length_starts"][mids]
    return q


# ------------------------------------------------------------------------------------------------------------------ rotations
def primary(cands: List[mf.Cand]):
    """(value, tol) of the first allowed candidate per row, and the rows where another allowed candidate differs beyond the bounds."""
    v0, t0, ok0 = cands[0]
    val, tol = torch.zeros_like(v0), torch.zeros_like(t0)
    seen = torch.zeros(ok0.shape, dtype=torch.bool, device=v0.device)
    amb = torch.zeros_like(seen)
    for v, t, ok in cands:
        ok = ok.expand(seen.shape)
        first = ok & ~seen
        amb = amb | (ok & seen & ((v - val).abs() > t + tol).any(-1))
        val = torch.where(first[..., None], v, val)
        tol = torch.where(first[..., None], t, tol)
        seen = seen | ok
    return val, tol, amb


def base_removed(q, tq, upright: bool):
    """base_rot_removed in float64: q (x) conj(0.5, 0.5, 0.5, 0.5) for a non-upright start, with its bound."""
    if upright:
        return q, tq
    b = torch.tensor(BASE_INV, dtype=q.dtype, device=q.device).expand_as(q)
    return mf.qmul(q, b), 0.5 * tq.sum(-1, keepdim=True).expand_as(tq) + mf.qmul8_err(q, b)


def heading_ref(q, tq, upright: bool):
    """The inverse heading of base_rot_removed(q): (hs, hc) of the heading angle in float64, its angle bound dth, and the rows where
    the heading is ill-conditioned (dth capped at 2 pi there, so any rotation passes)."""
    qb, tb_ = base_removed(q, tq, upright)
    x, y, z, w = qb.unbind(-1)
    rx = 2 * w * w - 1 + 2 * x * x
    ry = 2 * w * z + 2 * x * y
    n = torch.sqrt(rx * rx + ry * ry)
    dr = 4 * qb.abs().sum(-1) * tb_.amax(-1) + 8 * U32 * (1 + rx.abs() + ry.abs())
    ill = dr * 4 >= n
    dth = torch.where(ill, torch.full_like(n, 2 * math.pi), dr / torch.where(ill, torch.ones_like(n), n) + 16 * U32)
    th = torch.atan2(ry, rx)
    return torch.sin(0.5 * th), torch.cos(0.5 * th), dth, ill


def yaw_apply(hs, hc, dth, v, tv):
    """Rotation of v [..., 3] by the inverse heading (yaw_rot / my_quat_rotate with (0, 0, -hs, hc)) in float64, with its bound: the
    input bound mixed pairwise in xy, |v_xy| dth, 8 u32 |v| for the fp32 products and sums."""
    c = (hc * hc - hs * hs)[..., None]
    s = (2 * hs * hc)[..., None]
    x, y, zc = v[..., 0:1], v[..., 1:2], v[..., 2:3]
    out = torch.cat([c * x + s * y, c * y - s * x, zc], -1)
    vxy = torch.sqrt(x * x + y * y)
    vn = v.norm(dim=-1, keepdim=True)
    txy = tv[..., 0:1] + tv[..., 1:2] + vxy * dth[..., None] + 8 * U32 * vn
    return out, torch.cat([txy, txy, tv[..., 2:3] + 8 * U32 * zc.abs()], -1)


def yaw_qmul(hs, hc, dth, q, tq):
    """qmul((0, 0, -hs, hc), q) in float64 with its bound: pairwise mixing, |q| dth / 2, the 8-product rounding."""
    h = torch.stack([torch.zeros_like(hs), torch.zeros_like(hs), -hs, hc], -1)
    h = h.expand(q.shape)
    out = mf.qmul(h, q)
    pair = torch.stack([tq[..., 0] + tq[..., 1], tq[..., 0] + tq[..., 1], tq[..., 2] + tq[..., 3], tq[..., 2] + tq[..., 3]], -1)
    return out, pair + (0.5 * q.norm(dim=-1) * dth.expand(q.shape[:-1]))[..., None] + mf.qmul8_err(h, q)


def six_ref(q, tq):
    """quat_to_tan_norm (the rotated x and z axes) in the kernel's formula, float64, with its bound."""
    x, y, z, w = q.unbind(-1)
    s = 2 * w * w - 1
    out = torch.stack([s + 2 * x * x, 2 * (z * w + x * y), 2 * (-y * w + x * z), 2 * (y * w + x * z), 2 * (-x * w + y * z), s + 2 * z * z], -1)
    return out, (4 * q.abs().sum(-1) * tq.amax(-1) + 8 * U32 * (1 + q.abs().sum(-1) ** 2))[..., None].expand_as(out)


def expmap_six_cands(e, te) -> List[mf.Cand]:
    """quat_to_tan_norm(exp_map_to_quat(e)) of rows e [..., 3] known to within te [...] (Euclidean): the identity for |angle| <= 1e-5 and
    the rotation by |e| about e / |e| otherwise.  The general branch's bound: te (the columns of R(e) move by at most |de|), the angle's
    sqrt / wrap (atan2f of sinf, cosf) / sincosf roundings and the normalisations, (24 + 8 |e|) u32."""
    ang = e.norm(dim=-1)
    ident = torch.zeros(e.shape[:-1] + (6,), dtype=e.dtype, device=e.device)
    ident[..., 0] = 1.0
    ident[..., 5] = 1.0
    safe = torch.where(ang > 0, ang, torch.ones_like(ang))
    axis = e / safe[..., None]
    q = torch.cat([axis * torch.sin(0.5 * ang)[..., None], torch.cos(0.5 * ang)[..., None]], -1)
    six, _ = six_ref(q, torch.zeros_like(q))
    tol = (te + (24 + 8 * ang) * U32)[..., None].expand_as(six)
    lo, hi = ang * (1 - 2 * U32) - te, ang * (1 + 2 * U32) + te
    return [(ident, torch.zeros_like(ident), lo <= EXP_EPS32), (six, tol, hi > EXP_EPS32)]


# ------------------------------------------------------------------------------------------------------------------ AMP row
def amp_row_ref(p0, tp0, q0, tq0, v0, tv0, w0, tw0, dof, tdof, dvel, tdvel, key, tkey, upright: bool) -> Dict[str, object]:
    """build_amp_observations_smpl of the root state (p0 [n, 3], q0 [n, 4], v0, w0), the joints' exponential maps dof [n, 23, 3] with
    Euclidean bounds tdof [n, 23], dof velocities dvel [n, 69] and key-body positions key [n, 4, 3] (bodies 7, 3, 22, 17), float64 with
    bounds.  Returns {"h", "root", "vel", "ang", "dof_vel", "key"}: (ref, tol) over the row's columns, "dof_six": candidates [n, 19, 6],
    "ill": rows whose heading is ill-conditioned."""
    qb, tqb = base_removed(q0, tq0, upright)
    hs, hc, dth, ill = heading_ref(qb, tqb, True)
    rq, trq = yaw_qmul(hs, hc, dth, qb, tqb)
    out: Dict[str, object] = {"h": (p0[:, 2:3], tp0[:, 2:3]), "root": six_ref(rq, trq), "vel": yaw_apply(hs, hc, dth, v0, tv0),
                              "ang": yaw_apply(hs, hc, dth, w0, tw0), "ill": ill}
    kj = torch.tensor(KEPT_JOINTS, device=dof.device)
    out["dof_six"] = expmap_six_cands(dof[:, kj], tdof[:, kj])
    vi = (3 * kj[:, None] + torch.arange(3, device=dof.device)[None, :]).reshape(-1)
    out["dof_vel"] = (dvel[:, vi], tdvel[:, vi])
    rel = key - p0[:, None, :]
    trel = tkey + tp0[:, None, :] + U32 * rel.abs()
    k, tk = yaw_apply(hs[:, None], hc[:, None], dth[:, None], rel, trel)
    out["key"] = (k.reshape(len(p0), 12), tk.reshape(len(p0), 12))
    return out


AMP_COLS = {"h": (0, 1), "root": (1, 7), "vel": (7, 10), "ang": (10, 13), "dof_six": (13, 127), "dof_vel": (127, 184), "key": (184, 196)}


def check_amp(rep: Optional[Report], tag: str, got: torch.Tensor, ref: Dict[str, object], built: Optional[torch.Tensor] = None) -> None:
    """One AMP row per env, 196 or 195 floats, against amp_row_ref: each column group element-wise, the joints' rotation features by
    branch; the ill-conditioned share limited (outside `built`)."""
    width = got.shape[-1]
    skip = 196 - width
    n = got.shape[0]
    for name, (a, b) in AMP_COLS.items():
        if name == "h" and skip:
            continue
        g = got[:, a - skip:b - skip]
        if name == "dof_six":
            mf.check_branches(rep, f"{tag} amp dof six", g.reshape(n, 19, 6), ref["dof_six"])
        else:
            r, t = ref[name]
            if name in ("root", "vel", "ang", "key"):
                t = torch.where(ref["ill"][:, None], torch.full_like(t, math.inf), t)
            check(rep, f"{tag} amp {name}", g, r, t)
    limit_share(rep, f"{tag} amp heading", ref["ill"], built)


def limit_share(rep: Optional[Report], link: str, amb: torch.Tensor, built: Optional[torch.Tensor] = None,
                amb_max: float = AMBIGUOUS_MAX) -> float:
    """Records and limits the share of ambiguous rows outside `built`."""
    if built is not None:
        amb = amb & ~built
    share = float(amb.double().mean()) if amb.numel() else 0.0
    if rep is not None:
        rep.add(link + " (share)", 0.0, ambiguous=share)
    if not share < amb_max:
        raise BoundError(f"{link}: {share:.2e} of the rows are ambiguous (limit {amb_max})")
    return share


def motion_amp_ref(q: Dict[str, object], upright: bool) -> Dict[str, object]:
    """amp_row_ref of the un-fixed motion (rows k > 0): the gathered root, the primary slerp / exp-map candidates with their bounds."""
    pos, tpos = q["rg_pos"]
    vel, tvel = q["body_vel"]
    ang, tang = q["body_ang_vel"]
    rr, trr, amb_r = primary(mf.root_cands(q["rb_rot"]))
    dof, tdof, amb_d = primary(q["dof_pos"])
    dv, tdv = q["dof_vel"]
    kb = torch.tensor(KEY_BODIES, device=pos.device)
    ref = amp_row_ref(pos[:, 0], tpos[:, 0], rr, trr, vel[:, 0], tvel[:, 0], ang[:, 0], tang[:, 0], dof, tdof.norm(dim=-1), dv, tdv,
                      pos[:, kb], tpos[:, kb], upright)
    ref["ill"] = ref["ill"] | amb_r | amb_d.any(-1)
    return ref


def state_amp_ref(body: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, upright: bool) -> Dict[str, object]:
    """amp_row_ref of a written state (row 0, getup_amp_init): body [n, >= 24, 13], dof_pos / dof_vel [n, 69], all exact fp32."""
    b = f64(body)
    z = lambda t: torch.zeros_like(t)
    kb = torch.tensor(KEY_BODIES, device=b.device)
    dof = f64(dof_pos).reshape(len(b), 23, 3)
    return amp_row_ref(b[:, 0, 0:3], z(b[:, 0, 0:3]), b[:, 0, 3:7], z(b[:, 0, 3:7]), b[:, 0, 7:10], z(b[:, 0, 7:10]), b[:, 0, 10:13],
                       z(b[:, 0, 10:13]), dof, torch.zeros(dof.shape[:2], dtype=dof.dtype, device=dof.device), f64(dof_vel),
                       z(f64(dof_vel)), b[:, kb, 0:3], z(b[:, kb, 0:3]), upright)


# ------------------------------------------------------------------------------------------------------------------ reset state
def reset_state_ref(tb, mids: torch.Tensor, t0: torch.Tensor, floor: Optional[torch.Tensor], pose: str, upright: bool) -> Dict[str, object]:
    """The state reset_warps leaves for clips mids at t0 (teacher-forced on the exact rows): ground fix from floor[f0] (None: no fix, the
    reference-state reset), then the pose adjustment.  Returns (ref, tol) for "body_pos" / "body_vel" / "body_ang" [n, B, 3],
    "root_pos" / "root_vel" / "root_ang" [n, 3], "dof_vel" [n, 3(B-1)]; candidates for "body_rot" [n, B, 4], "root_rot" [n, 4] and
    "dof_pos" [n, B-1, 3]; "amb" rows (ill-conditioned heading or an ambiguous root rotation); the query "q"."""
    q = motion_ref(tb, mids, t0)
    pos, tpos = (x.clone() for x in q["rg_pos"])
    if floor is not None:
        fl = f64(floor)[q["f0"]]
        rz, trz = pos[:, 0, 2].clone(), tpos[:, 0, 2].clone()
        s = fl + rz
        d = s - GROUND_MARGIN
        pz = pos[..., 2] - d[:, None]
        tpos[..., 2] = tpos[..., 2] + (trz + U32 * (s.abs() + d.abs() + GROUND_MARGIN))[:, None] + U32 * pz.abs()
        pos[..., 2] = pz
    vel, tvel = q["body_vel"]
    ang, tang = q["body_ang_vel"]
    rot = q["rb_rot"]
    rr, trr, amb = primary(mf.root_cands(rot))
    out: Dict[str, object] = {"q": q, "dof_pos": q["dof_pos"], "dof_vel": q["dof_vel"]}
    if pose == POSE_FACE_X:
        hs, hc, dth, ill = heading_ref(rr, trr, upright)
        amb = amb | ill
        rp, trp = pos[:, 0:1], tpos[:, 0:1]
        rel = pos - rp
        trel = tpos + trp + U32 * rel.abs()
        pr, tpr = yaw_apply(hs[:, None], hc[:, None], dth[:, None], rel, trel)
        pos, tpos = pr + rp, tpr + trp + U32 * (pr + rp).abs()
        vel, tvel = yaw_apply(hs[:, None], hc[:, None], dth[:, None], vel, tvel)
        rot = [yaw_qmul(hs[:, None], hc[:, None], dth[:, None], v, t) + (ok,) for v, t, ok in rot]
        # humanoid_speed.py turns the root's angular velocity but leaves the bodies' (body_ang_vel) as sampled
        root_ang = yaw_apply(hs, hc, dth, ang[:, 0], tang[:, 0])
    else:
        root_ang = (ang[:, 0], tang[:, 0])
    out.update(body_pos=(pos, tpos), body_vel=(vel, tvel), body_ang=(ang, tang), body_rot=rot, root_rot=mf.root_cands(rot), amb=amb)
    root_pos, troot = pos[:, 0].clone(), tpos[:, 0].clone()
    if pose == POSE_ROOT_XY_ZERO:
        root_pos[:, :2] = 0.0
        troot[:, :2] = 0.0
    out.update(root_pos=(root_pos, troot), root_vel=(vel[:, 0], tvel[:, 0]), root_ang=root_ang)
    return out


def check_state(rep: Optional[Report], tag: str, got: Dict[str, torch.Tensor], ref: Dict[str, object], built=None) -> None:
    """The written state of the reset envs against reset_state_ref: got has "body" [n, B, 13], "root" [n, 13], "dof_pos" / "dof_vel"
    [n, 3(B-1)].  Rows in ref["amb"] pass any rotation-dependent value; their share is limited."""
    body, root = got["body"], got["root"]
    n, B = body.shape[0], body.shape[1]
    amb = ref["amb"]
    loose = lambda t, m: torch.where(m.reshape(m.shape + (1,) * (t.dim() - 1)), torch.full_like(t, math.inf), t)
    for name, sl, key in (("body pos", slice(0, 3), "body_pos"), ("body vel", slice(7, 10), "body_vel"), ("body ang", slice(10, 13), "body_ang")):
        r, t = ref[key]
        check(rep, f"{tag} {name}", body[..., sl], r, loose(t, amb))
    for name, sl, key in (("root pos", slice(0, 3), "root_pos"), ("root vel", slice(7, 10), "root_vel"), ("root ang", slice(10, 13), "root_ang")):
        r, t = ref[key]
        check(rep, f"{tag} {name}", root[:, sl], r, loose(t, amb))
    rc = [(v, t, ok | amb[:, None]) for v, t, ok in ref["body_rot"]]
    mf.check_branches(rep, f"{tag} body rot", body[..., 3:7], rc, built=amb[:, None] if built is None else (amb | built)[:, None])
    rr = [(v, t, ok | amb) for v, t, ok in ref["root_rot"]]
    mf.check_branches(rep, f"{tag} root rot", root[:, 3:7], rr, built=amb if built is None else amb | built)
    mf.check_branches(rep, f"{tag} dof pos", got["dof_pos"].reshape(n, B - 1, 3), ref["dof_pos"], built=None if built is None else built[:, None])
    check(rep, f"{tag} dof vel", got["dof_vel"], *ref["dof_vel"])
    limit_share(rep, f"{tag} heading / root branch", amb, built)


# ------------------------------------------------------------------------------------------------------------------ strike, task
def strike_ref(u: torch.Tensor, root_xy: torch.Tensor, near_prob: float, near_dist: float, dmin: float, dmax: float) -> Dict[str, tuple]:
    """_reset_target of the strike task for uniforms u [n, 4] (near, distance, bearing, yaw) around root_xy [n, 2] (exact, 0 after
    ROOT_XY_ZERO): (ref, tol) of the target's xy [n, 2] and of its yaw quaternion's z, w [n, 2]; the near decision is exact."""
    u = f64(u)
    f = lambda x: float(np.float32(x))
    near = u[:, 0] < f(near_prob)
    dm = torch.where(near, torch.full_like(u[:, 0], f(near_dist)), torch.full_like(u[:, 0], f(dmax)))
    span = dm - f(dmin)
    dist = span * u[:, 1] + f(dmin)
    tdist = U32 * (span.abs() + (span * u[:, 1]).abs() + dist.abs())
    th, yaw = 2 * math.pi * u[:, 2], 2 * math.pi * u[:, 3]
    dth = abs(TWO_PI32 - 2 * math.pi) * u[:, 2] + U32 * th + 4 * U32
    dyaw = 0.5 * (abs(TWO_PI32 - 2 * math.pi) * u[:, 3] + U32 * yaw) + 4 * U32
    xy = torch.stack([dist * torch.cos(th), dist * torch.sin(th)], 1)
    txy = tdist[:, None] + dist[:, None] * dth[:, None] + U32 * (2 * xy.abs() + (xy + f64(root_xy)).abs())
    zw = torch.stack([torch.sin(0.5 * yaw), torch.cos(0.5 * yaw)], 1)
    return {"xy": (xy + f64(root_xy), txy), "zw": (zw, dyaw[:, None].expand_as(zw).clone())}


def task_ref(kind: str, rand: torch.Tensor, steps: torch.Tensor, progress: torch.Tensor, dist_max: float, height_min: float,
             height_max: float, speed_min: float, speed_max: float) -> Dict[str, tuple]:
    """_reset_task of reach (target [n, 3]) or speed (target speed [n]), float64 with the bound of its fp32 operations; change_steps
    exact."""
    f = lambda x: float(np.float32(x))
    u = f64(rand)
    if kind == "reach":
        xy = f(dist_max) * (2 * u[:, :2] - 1)
        hs = f(f(height_max) - f(height_min))
        z = hs * u[:, 2:3] + f(height_min)
        v = torch.cat([xy, z], 1)
        t = torch.cat([U32 * (xy.abs() + f(dist_max) * (2 * u[:, :2]).abs()),
                       U32 * ((hs * u[:, 2:3]).abs() + z.abs())], 1)
    else:
        sc = f(f(speed_max) - f(speed_min))
        v = sc * u[:, 0] + f(speed_min)
        t = U32 * ((sc * u[:, 0]).abs() + v.abs())
    return {"target": (v, t), "change_steps": progress.long() + steps.long()}


# ------------------------------------------------------------------------------------------------------------------ terrain spawn
def spawn_ref(state: Dict[str, object], loc: torch.Tensor, coord_x: torch.Tensor, coord_y: torch.Tensor, hf: torch.Tensor, hscale: float,
              vscale: float, points: torch.Tensor, upright: bool, root_rot: torch.Tensor) -> Dict[str, object]:
    """The terrain spawn on reset_state_ref's (AS_IS, ground-fixed) state: root xy = the table entry, bodies shifted in xy (z not lifted),
    root z lifted by the mean center height at the new xy.  The center points turn with the kernel's own root rotation `root_rot`
    [n, 4] (what it wrote, checked by the root rot link), so their bound is that of the fp32 yaw and point arithmetic alone.  A point
    within its bound of a cell edge takes the lowest and highest height its cells can give; the root z is checked against that interval
    and the row counted ambiguous."""
    dev = hf.device
    nx, ny = coord_x[loc].float(), coord_y[loc].float()
    pos, tpos = state["body_pos"]
    rp, trp = pos[:, 0], tpos[:, 0]
    dx = torch.stack([f64(nx) - rp[:, 0], f64(ny) - rp[:, 1]], 1)
    bxy = pos[..., :2] + dx[:, None, :]
    tb_ = tpos[..., :2] + trp[:, None, :2] + U32 * (dx.abs()[:, None, :] + bxy.abs())
    body_pos = torch.cat([bxy, pos[..., 2:3]], -1)
    body_tol = torch.cat([tb_, tpos[..., 2:3]], -1)
    # the yaw of yaw_only(base_rot_removed(root rot)): angle 2 atan2(z, w), bound 2 (tz + tw) / |(z, w)| plus the roundings
    rr = f64(root_rot).to(dev)
    qb, tqb = base_removed(rr, torch.zeros_like(rr), upright)
    nz = torch.sqrt(qb[:, 2] ** 2 + qb[:, 3] ** 2)
    phi = 2 * torch.atan2(qb[:, 2], qb[:, 3])
    ill = (tqb[:, 2] + tqb[:, 3]) * 4 >= nz
    dphi = torch.where(ill, torch.full_like(nz, 2 * math.pi), 2 * (tqb[:, 2] + tqb[:, 3]) / torch.where(ill, torch.ones_like(nz), nz) + 8 * U32)
    pts = f64(points).to(dev)
    c, s = torch.cos(phi)[:, None], torch.sin(phi)[:, None]
    rx = c * pts[None, :, 0] - s * pts[None, :, 1]
    ry = s * pts[None, :, 0] + c * pts[None, :, 1]
    # the fp32 rotated offset is within dr of (rx, ry) (quat_apply_rn: 12 u32 |off|); the world point is its round-to-nearest sum with
    # the fp32 root xy, so it lies between the roundings of the two ends
    dr = pts[:, :2].norm(dim=-1)[None, :] * (dphi[:, None] + 12 * U32)
    h32 = torch.tensor(hscale, dtype=torch.float32)
    R, Cc = hf.shape
    hfi = hf.long()

    def cells(origin, r, top):
        lo, hi = (f64(origin)[:, None] + r - dr).float(), (f64(origin)[:, None] + r + dr).float()
        # fp32 quotients through float64 (innocuous double rounding), on any device: CUDA divides by a scalar with its reciprocal
        q = lambda x: (x.double() / float(h32)).float().long().clamp(0, top)
        return q(lo), q(hi)

    pxa, pxb = cells(nx, rx, R - 2)
    pya, pyb = cells(ny, ry, Cc - 2)
    hts = []
    for px in (pxa, pxb):
        for py in (pya, pyb):
            hts.append(torch.minimum(hfi[px, py], hfi[px + 1, py + 1]).float() * torch.tensor(vscale, dtype=torch.float32))
    hts = torch.stack(hts, -1).double()
    edge = ((pxa != pxb) | (pya != pyb)).any(-1) | ill
    P = pts.shape[0]
    lo, hi = hts.amin(-1).sum(-1) / P, hts.amax(-1).sum(-1) / P
    tmean = 5 * U32 * hts.abs().amax(-1).sum(-1) / P + U32 * hi.abs()
    rz, trz = rp[:, 2], trp[:, 2]
    z_lo, z_hi = rz + lo, rz + hi
    root_pos = torch.stack([f64(nx), f64(ny), 0.5 * (z_lo + z_hi)], 1)
    root_tol = torch.stack([torch.zeros_like(rz), torch.zeros_like(rz), 0.5 * (z_hi - z_lo) + trz + tmean + U32 * z_hi.abs()], 1)
    return {"body_pos": (body_pos, body_tol), "root_pos": (root_pos, root_tol), "edge": edge}


# ------------------------------------------------------------------------------------------------------------------ getup, exact
def getup_ref(cands: torch.Tensor, terminate: torch.Tensor, avail: torch.Tensor, assign: torch.Tensor, recovery_u: torch.Tensor,
              fall_u: torch.Tensor, key_bits: torch.Tensor, recovery_prob: float, fall_prob: float, recovery_steps: int,
              counter: torch.Tensor) -> Dict[str, torch.Tensor]:
    """getup_classify / keys / select / apply on CPU tensors: cands the ascending reset envs, draws per env (indexed by env), key_bits
    per state.  Returns the lists, counts, the error increment, fall_pick, and the updated avail / assign / counter."""
    avail, assign, counter = avail.clone(), assign.clone(), counter.clone()
    avail[assign[cands]] = 0
    free = int((avail == 0).sum())
    rec = (recovery_u[cands] < np.float32(recovery_prob)) & (terminate[cands] == 1)
    want = ~rec & (fall_u[cands] < np.float32(fall_prob))
    fpos = torch.cumsum(want.long(), 0) - 1
    fall = want & (fpos < free)
    ref = ~rec & ~fall
    falls = min(int(want.sum()), free)
    counter[cands] = torch.where(ref, torch.zeros_like(counter[cands]), torch.full_like(counter[cands], recovery_steps))
    free_ids = (avail == 0).nonzero().flatten()
    order = free_ids[torch.argsort(key_bits[free_ids].long(), stable=True)]   # (key bits, id): free_ids ascend, the sort is stable
    pick = order[:falls]
    fall_list = cands[fall]
    avail[pick] = 1
    assign[fall_list] = pick
    return {"env_list": cands, "ref_list": cands[ref], "fall_list": fall_list, "recovery_list": cands[rec],
            "class_counts": torch.tensor([int(ref.sum()), falls, int(rec.sum())], dtype=torch.int32), "error": int(want.sum()) - falls,
            "fall_pick": pick, "avail": avail, "assign": assign, "counter": counter,
            "env_class": torch.where(ref, 1, torch.where(fall, 2, 3))}      # PULSE_GETUP_REF / _FALL / _RECOVERY


# ------------------------------------------------------------------------------------------------------------------ trajectories
def traj_ref(start: torch.Tensor, draws: torch.Tensor, dtheta_scale: float, dspeed_scale: float, seg_dt: float, speed_min: float,
             speed_max: float, sharp_turn_prob: float) -> Dict[str, torch.Tensor]:
    """TrajGenerator.reset of start xy [n, 2] (fp32) with draws [n, 4 S + 2] (CPU): "xy" (ref, tol) [n, S + 1, 2] of the waypoints."""
    f = lambda x: torch.tensor(float(np.float32(x)), dtype=torch.float32)
    S = TRAJ_SEGS
    u = draws.float().cpu()
    x0, y0 = start[:, 0].float().cpu(), start[:, 1].float().cpu()
    pi = f(3.14159265358979)
    smin, smax, dths, dsps, segdt, p = f(speed_min), f(speed_max), f(dtheta_scale), f(dspeed_scale), f(seg_dt), f(sharp_turn_prob)
    n = len(u)
    ang = torch.zeros(n, dtype=torch.float64)
    px, py = f64(x0), f64(y0)
    tx, ty = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    xs, ys, txs, tys = [px.clone()], [py.clone()], [tx.clone()], [ty.clone()]
    speed = torch.zeros(n, dtype=torch.float32)
    for k in range(S):
        if k == 0:
            dth = pi * (2.0 * u[:, 4 * S] - 1.0)
            speed = (smax - smin) * u[:, 4 * S + 1] + smin
        else:
            sharp = u[:, 2 * S + k] < p
            dth = torch.where(sharp, pi * (2.0 * u[:, S + k] - 1.0), (2.0 * u[:, k] - 1.0) * dths)
            speed = torch.minimum(torch.maximum(speed + (2.0 * u[:, 3 * S + k] - 1.0) * dsps, smin), smax)
        ang = ang + dth.double()
        th = f64(ang.float())
        seg = f64(speed * segdt)
        dx, dy = torch.cos(th) * seg, -torch.sin(th) * seg
        tx = tx + 4 * U32 * seg + U32 * dx.abs()
        ty = ty + 4 * U32 * seg + U32 * dy.abs()
        if k == 0:
            tx, ty = tx + U32 * (dx + px).abs(), ty + U32 * (dy + py).abs()
        px, py = px + dx, py + dy
        xs.append(px.clone())
        ys.append(py.clone())
        txs.append(tx + U32 * px.abs())
        tys.append(ty + U32 * py.abs())
    return {"xy": (torch.stack([torch.stack(xs, 1), torch.stack(ys, 1)], -1), torch.stack([torch.stack(txs, 1), torch.stack(tys, 1)], -1))}


def check_traj(rep: Optional[Report], tag: str, verts: torch.Tensor, start: torch.Tensor, ref: Dict[str, torch.Tensor]) -> None:
    """Waypoints [n, S + 1, 3]: the start xy and every z exactly, the xy against traj_ref."""
    v = verts.cpu()
    check_exact(rep, f"{tag} traj start", v[:, 0, :2], start.cpu())
    check_exact(rep, f"{tag} traj z", v[..., 2], torch.zeros(v.shape[:2]))
    check(rep, f"{tag} traj verts", v[..., :2], *ref["xy"])
