"""Teacher-forced float64 references of the motion library's kernels, each with an element-wise bound derived from the fp32 operations
its kernel performs (the style of tests/fp64_ref.py: BoundError names the link, a Report keeps the margins).

Links and what feeds them:
* loader pose pass (motion_loader.cu, one thread per frame): `grs` and `lrs` from the on-disk float64 clips; `gts` by forward kinematics
  in float64 from the kernel's own fp32 `lrs`.  The kernel does the heading step and the local rotations in float64 and rounds once, so
  their bound is one fp32 rounding plus 64 u64.  FK runs in fp32: the bound of a body's rotation grows by 13 u32 per joint of the chain
  (the 16-product Hamilton form, 4 u32 per component, and the normalisation), its position by the parent's rotation error times 2 |offset|,
  14 u32 |offset| for the two products of quat_rotate and one rounding per add.
* loader velocity pass: `tmp_vel` = np.gradient of the kernel's `gts` over the clip's own dt (one-sided at clip ends, 0 for a clip's only
  frame); `tmp_ang` from consecutive heading-rotated global rotations of the on-disk clip (last frame 0) with the angle in the
  well-conditioned form 2 atan2(|v|, w).  The kernel's acos(2 w^2 - 1) in float64 is conditioned as 1 / sin(angle) and, near angle 0,
  as sqrt(2 delta): both enter its bound with delta = 132 u64 (the float64 quaternion pipeline moves w by at most 32 u64).
  `dvs` from the kernel's fp32 `lrs` pair (f, f + 1), the last frame repeating the pair (f - 1, f): the bound of the kernel's 8-product
  quat_mul is computed from its own intermediate values (qmul8_err), then carried through the exponential map, so it is tight except
  where the rotation between the two frames is near zero (the fp32 1 - w^2 cancels).
* loader filter pass: a 17-tap sigma = 2 gaussian, normalised in float64, `nearest` inside the clip, on the kernel's own `tmp_vel` /
  `tmp_ang`.  fp32: expf (2 ulp), the 9-term weight sum (8 u32), the quotient, 17 fused multiply-adds: 32 u32 sum |w x|.
* packing: the frame and aux records equal the tables bit for bit, pads zero.
* query (motion_state_kernel, smplx_motion_state_kernel): frame indices and blend are fp32 arithmetic in the reference's order, compared
  exactly with oracle.pulse_oracle.frame_blend.  With the kernel's blend as the operand: the lerps (three roundings, one more for the
  offset), the reference's piecewise slerp, and the exponential map of the slerped local rotations.

Choices:
* Frame rates: the kernel receives fp32 fps (loader) or fp32 dt (query); the references follow the clip's float64 rate, as the reference
  implementation does, and every bound that divides by dt carries one more u32 relative for the rate's rounding.
* slerp follows torch_utils.slerp, branches included: c >= 1 returns q0, s = sqrt(1 - c^2) < 0.001 returns the midpoint whatever t is.
  The exponential map follows quat_to_exp_map: s = sqrt(1 - w^2) <= 1e-5 gives 0, angles 2 acos(w) past pi wrap to angle - 2 pi.  The fp32
  kernel decides each branch on values within a bound of the float64 ones: the dot product c within 5 u32 sum |a b|, s^2 within
  2 |c| dc + dc^2 + u32, the angle within its conditioning.  A row whose float64 value lies within that bound of a threshold may take either
  branch: every branch it can take is a candidate, the row passes if one candidate holds it, and the share of such rows is reported as
  ambiguous.  Outside the rows a test builds on a threshold the share must stay under AMBIGUOUS_MAX.
* Inside the general slerp branch the weights sin((1 - t) h) / s are insensitive to the error of h (|d/dh| <= 0.25 h on [0, pi/2], checked
  in test_motion_fp64_cpu), but the fp32 s = sqrt(1 - c^2) carries u32 / (2 s^2) relative from the rounding of c^2: 3 % at s = 0.001.  That
  is the real conditioning of the reference's formula in fp32, and the bound keeps it.
"""
import math
from typing import Dict, List, Optional, Tuple

import torch

from tests.fp64_ref import U32, U64, BoundError, Report, check, check_exact, f64  # noqa: F401  (re-exported for the tests)

AMBIGUOUS_MAX = 1e-3
PI32 = float(torch.tensor(math.pi, dtype=torch.float32))         # 3.14159274: the kernel's wrap threshold
TWO_PI32 = float(torch.tensor(2 * math.pi, dtype=torch.float32))
RADIUS = 8                                                       # gaussian_filter1d(sigma = 2, truncate = 4)
SLERP_MID = 0.001
EXP_EPS = 1e-5
FRAME_REC, AUX_REC = 312, 240
SMPLX_FRAME_REC, SMPLX_AUX_REC = 676, 364

Cand = Tuple[torch.Tensor, torch.Tensor, torch.Tensor]          # (value [..., C], tol [..., C], allowed [...])


# ------------------------------------------------------------------------------------------------------------------ float64 algebra
def qmul(a, b):
    """Hamilton product, xyzw."""
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                        aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], -1)


def qconj(q):
    return torch.cat([-q[..., :3], q[..., 3:]], -1)


def qnormalize(q):
    """poselib quat_normalize: w >= 0, unit length."""
    q = torch.where(q[..., 3:] < 0, -q, q)
    return q / q.norm(dim=-1, keepdim=True).clamp_min(1e-9)


def qrotate(q, v):
    """Imaginary part of q (x) (v, 0) (x) conj(q) (poselib quat_rotate; scales by |q|^2 for a non-unit q, as the kernel does)."""
    return qmul(qmul(q, torch.cat([v, torch.zeros_like(v[..., :1])], -1)), qconj(q))[..., :3]


def qmul8_err(a, b):
    """Bound of the fp32 error of quat_math.cuh's 8-product quat_mul on fp32 operands a, b (float64 tensors holding fp32 values): every
    rounding bounded by u32 |its result| and carried to the output with its coefficient (1, or 0.5 through qq)."""
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    prod = lambda s, t: (s * t, 3 * U32 * (s * t).abs())          # two rounded sums, one rounded product
    ww, eww = prod(az + ax, bx + by)
    yy, eyy = prod(aw - ay, bw + bz)
    zz, ezz = prod(aw + ay, bw - bz)
    xx = ww + yy + zz
    exx = eww + eyy + ezz + U32 * ((ww + yy).abs() + xx.abs())
    p5, e5 = prod(az - ax, bx - by)
    qq = 0.5 * (xx + p5)
    eqq = 0.5 * (exx + e5 + U32 * (xx + p5).abs())
    out = []
    for base, ebase, (s, t) in ((ww, eww, (az - ay, by - bz)), (xx, exx, (ax + aw, bx + bw)), (yy, eyy, (aw - ax, by + bz)),
                                (zz, ezz, (az + ay, bw - bx))):
        p, ep = prod(s, t)
        r = qq - base + p
        out.append(eqq + ebase + ep + U32 * ((qq - base).abs() + r.abs()))
    w, x, y, z = out
    return torch.stack([x, y, z, w], -1)


def _acos_err(c, dc):
    """max |acos(c') - acos(c)| over |c' - c| <= dc: the slope 1 / sqrt(1 - c^2) away from +-1, sqrt(2 dc) (times 1.1) at the ends."""
    m = torch.sqrt(torch.clamp(1.0 - (c.abs() + dc) ** 2, min=0.0))
    slope = torch.where(m > 0, dc / torch.where(m > 0, m, torch.ones_like(m)), torch.full_like(m, math.inf))
    return torch.minimum(slope, 1.1 * torch.sqrt(2.0 * dc))


# ------------------------------------------------------------------------------------------------------------------ comparators
def check_branches(rep: Optional[Report], link: str, got: torch.Tensor, cands: List[Cand], built: Optional[torch.Tensor] = None,
                   amb_max: float = AMBIGUOUS_MAX) -> Tuple[float, float]:
    """got [..., C] against branch candidates: a row (all of its C components) passes if one allowed candidate holds it element-wise.
    Rows with more than one allowed candidate are ambiguous; outside `built` (rows a test put on a threshold) their share must stay under
    amb_max.  Returns (largest err / tol of the best candidate per row, ambiguous share)."""
    g = f64(got)
    rows = g.shape[:-1]
    best = torch.full(rows, math.inf, dtype=torch.float64, device=g.device)
    n_ok = torch.zeros(rows, dtype=torch.int64, device=g.device)
    first_v = torch.zeros_like(g)
    first_t = torch.zeros_like(g)
    amb_rows = torch.zeros(rows, dtype=torch.bool, device=g.device)
    for ref, tol, ok in cands:
        if ref.shape != g.shape:
            raise BoundError(f"{link}: shape {tuple(g.shape)} vs reference {tuple(ref.shape)}")
        err = (g - ref).abs()
        r = torch.where(tol > 0, err / torch.where(tol > 0, tol, torch.ones_like(tol)),
                        torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
        r = torch.where(torch.isnan(err), torch.full_like(err, math.nan), r).amax(-1)
        ok = ok.expand(rows)
        best = torch.where(ok, torch.minimum(best, r), best)
        # ambiguous: a second allowed branch whose value the first allowed one's bound does not cover
        differs = ((ref - first_v).abs() > tol + first_t).any(-1)
        amb_rows = amb_rows | (ok & (n_ok > 0) & differs)
        first = ok & (n_ok == 0)
        first_v = torch.where(first[..., None], ref, first_v)
        first_t = torch.where(first[..., None], tol, first_t)
        n_ok = n_ok + ok.long()
    if bool((n_ok == 0).any()):
        raise BoundError(f"{link}: a row has no candidate branch (reference bug)")
    if built is not None:
        amb_rows = amb_rows & ~built.expand(rows)
    amb = float(amb_rows.double().mean()) if amb_rows.numel() else 0.0
    worst = float(best.max()) if best.numel() else 0.0
    if rep is not None:
        rep.add(link, worst, ambiguous=amb)
    if not worst < 1.0:
        k = int(torch.nan_to_num(best, nan=math.inf).reshape(-1).argmax())
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(k), rows))
        vals = [f"{float(c[0].reshape(-1, g.shape[-1])[k].abs().max()):.3e}" for c in cands]
        raise BoundError(f"{link}: err/tol {worst:.3f} at row {idx}: got {g.reshape(-1, g.shape[-1])[k].tolist()}, "
                         f"{int(n_ok.reshape(-1)[k])} allowed branch(es); candidate magnitudes {vals}")
    if not amb < amb_max:
        raise BoundError(f"{link}: {amb:.2e} of the rows lie within the bound of a branch decision (limit {amb_max})")
    return worst, amb


# ------------------------------------------------------------------------------------------------------------------ loader
def _headed(quat, frame_clip, headings):
    """The heading step: R_z(h) (x) normalize(q) per frame (none without headings: the on-disk rotations as they are)."""
    q = f64(quat)
    if headings is None:
        return q
    h = f64(headings)[frame_clip.long()]
    r = torch.stack([torch.zeros_like(h), torch.zeros_like(h), torch.sin(0.5 * h), torch.cos(0.5 * h)], -1)[:, None, :]
    return qmul(r.expand_as(q), q / q.norm(dim=-1, keepdim=True))


def loader_pose_ref(quat, trans, frame_clip, headings, parents, local_translation, lrs_k) -> Dict[str, tuple]:
    """grs, lrs from the on-disk clips; gts by float64 FK from the kernel's lrs_k [F, J, 4].  Returns {name: (ref, tol)}; "lrs" also
    carries a mask of rows whose w is within the float64 bound of 0 (the w >= 0 flip may go either way)."""
    g = _headed(quat, frame_clip, headings)
    F, J = g.shape[0], g.shape[1]
    out = {"grs": (g, U32 * g.abs() + 64 * U64 * (1 + g.abs()))}
    lr = torch.empty_like(g)
    for j, p in enumerate(parents):
        lr[:, j] = g[:, j] if p < 0 else qnormalize(qmul(qconj(g[:, p]), g[:, j]))
    raw_w = torch.stack([torch.ones_like(g[:, 0, 3]) if p < 0 else qmul(qconj(g[:, p]), g[:, j])[..., 3] for j, p in enumerate(parents)], 1)
    out["lrs"] = (lr, U32 * lr.abs() + 64 * U64 * (1 + lr.abs()), raw_w.abs() <= 64 * U64)
    # forward kinematics in float64 on the kernel's fp32 local rotations
    l = f64(lrs_k)
    loc = f64(local_translation)
    t = f64(trans)
    if headings is not None:
        h = f64(headings)[frame_clip.long()]
        c, s = torch.cos(h), torch.sin(h)
        t = torch.stack([c * t[:, 0] - s * t[:, 1], s * t[:, 0] + c * t[:, 1], t[:, 2]], -1)
    rot, pos = [None] * J, [None] * J
    e_rot = [None] * J
    e_pos = [None] * J
    for j, p in enumerate(parents):
        if p < 0:
            rot[j], pos[j] = l[:, j], t
            e_rot[j] = torch.zeros(F, dtype=torch.float64, device=l.device)
            e_pos[j] = U32 * t.abs() + 16 * U64 * (1 + t.abs())
        else:
            rot[j] = qnormalize(qmul(rot[p], l[:, j]))
            qn2 = (rot[p] * rot[p]).sum(-1)
            off = qrotate(rot[p], loc[j].expand(F, 3))
            pos[j] = off + pos[p]
            ln = float(loc[j].norm())
            e_rot[j] = e_rot[p] * l[:, j].norm(dim=-1) + 13 * U32
            e_pos[j] = e_pos[p] + ((2 * e_rot[p] * qn2.sqrt() + 14 * U32 * qn2) * ln)[:, None] + U32 * (off.abs() + pos[j].abs())
    out["gts"] = (torch.stack(pos, 1), torch.stack(e_pos, 1))
    return out


def clip_bounds(frame_clip, clip_start):
    """[f0, f1) of every frame's clip."""
    c = frame_clip.long()
    cs = clip_start.long()
    return cs[c], cs[c + 1]


def loader_velocity_ref(gts_k, lrs_k, quat, frame_clip, clip_start, fps, headings) -> Dict[str, tuple]:
    """tmp_vel from the kernel's gts, tmp_ang from the on-disk rotations, dvs from the kernel's lrs.  fps: the clips' float64 rates.
    Returns {"tmp_vel": (ref, tol), "tmp_ang": (ref, tol), "dvs": candidates}."""
    dev = gts_k.device
    F = gts_k.shape[0]
    f = torch.arange(F, device=dev)
    f0, f1 = clip_bounds(frame_clip, clip_start)
    r = f64(fps)[frame_clip.long()]                                 # the clip's own rate
    dt = 1.0 / r
    fa = torch.where(f > f0, f - 1, f)
    fb = torch.where(f + 1 < f1, f + 1, f)
    gk = f64(gts_k)
    span = (fb - fa).double()
    diff = gk[fb] - gk[fa]
    v = torch.where((span > 0)[:, None, None], diff / torch.where(span > 0, span * dt, torch.ones_like(dt))[:, None, None], torch.zeros_like(diff))
    # the fp32 difference, the rate's rounding, the cast of (fb - fa) dt, the reciprocal and the product: one u32 each
    out = {"tmp_vel": (v, 6 * U32 * v.abs())}
    # angular velocity from consecutive headed global rotations, float64
    g = _headed(quat, frame_clip, headings)
    has_next = f + 1 < f1
    nxt = torch.where(has_next, f + 1, f)
    d = qnormalize(qmul(g[nxt], qconj(g)))
    vn = d[..., :3].norm(dim=-1)
    ang = 2.0 * torch.atan2(vn, d[..., 3])
    w = d[..., :3] / vn.clamp_min(1e-9)[..., None] * (ang / dt[:, None])[..., None]
    w = torch.where(has_next[:, None, None], w, torch.zeros_like(w))
    delta = 132 * U64
    e_ang = _acos_err(torch.cos(ang), torch.full_like(ang, delta)) + 4 * U64 * ang
    tol = U32 * w.abs() + ((e_ang + 128 * U64) * r[:, None])[..., None] + (U32 + 8 * U64) * w.abs()
    out["tmp_ang"] = (w, torch.where(has_next[:, None, None], tol, torch.zeros_like(tol)))
    # dof velocities, joints 1..J-1, from the kernel's local rotations: pair (fs, fs + 1), fs = f or f - 1 at the clip's last frame
    fs = torch.where(f + 1 < f1, f, f - 1)
    pair = (fs >= f0) & (fs + 1 < f1)
    fs_c = torch.where(pair, fs, f)
    fs1 = torch.where(pair, fs + 1, f)
    l0, l1 = qconj(f64(lrs_k[:, 1:]))[fs_c], f64(lrs_k[:, 1:])[fs1]
    dq = qmul(l0, l1)
    cands = []
    rr = r[:, None, None]
    for e, t, ok in expmap_cands(dq, qmul8_err(l0, l1)):
        ok = ok & pair[:, None]
        cands.append((e * rr, t * rr + 3 * U32 * (e * rr).abs(), ok))
    zero = torch.zeros_like(dq[..., :3])
    cands.append((zero, zero, (~pair)[:, None].expand(dq.shape[:-1])))
    out["dvs"] = cands
    return out


def gaussian_weights(device=None) -> torch.Tensor:
    k = torch.arange(-RADIUS, RADIUS + 1, dtype=torch.float64, device=device)
    w = torch.exp(-0.5 * k * k / 4.0)
    return w / w.sum()


def filter_taps(frame_clip, clip_start) -> torch.Tensor:
    """[F, 17] source frames of the `nearest` filter, clamped to each frame's own clip."""
    F = frame_clip.shape[0]
    f = torch.arange(F, device=frame_clip.device)
    f0, f1 = clip_bounds(frame_clip, clip_start)
    t = f[:, None] + torch.arange(-RADIUS, RADIUS + 1, device=f.device)[None, :]
    return torch.minimum(torch.maximum(t, f0[:, None]), f1[:, None] - 1)


def loader_filter_ref(tmp_vel_k, tmp_ang_k, frame_clip, clip_start) -> Dict[str, tuple]:
    w = gaussian_weights(tmp_vel_k.device)
    taps = filter_taps(frame_clip, clip_start)
    out = {}
    for name, x in (("gvs", tmp_vel_k), ("gavs", tmp_ang_k)):
        terms = w[None, :, None, None] * f64(x)[taps]                  # [F, 17, J, 3]
        out[name] = (terms.sum(1), 32 * U32 * terms.abs().sum(1))
    return out


# ------------------------------------------------------------------------------------------------------------------ packing
def packed_records(tb, smplx: bool = False):
    """The frame and aux records the pack kernels must write, bit for bit (float32)."""
    F = tb["gts"].shape[0]
    fr = torch.cat([tb["gts"].reshape(F, -1), tb["grs"].reshape(F, -1), tb["gvs"].reshape(F, -1), tb["gavs"].reshape(F, -1)], 1).float()
    parts = [tb["lrs"].reshape(F, -1), tb["dvs"].reshape(F, -1)]
    if not smplx:
        parts.append(tb["motion_aa"].reshape(F, -1))
    ax = torch.cat(parts, 1).float()
    width = SMPLX_AUX_REC if smplx else AUX_REC
    ax = torch.cat([ax, torch.zeros(F, width - ax.shape[1], dtype=ax.dtype, device=ax.device)], 1)
    return fr, ax


# ------------------------------------------------------------------------------------------------------------------ query
def lerp_ref(p0, p1, b, offset=None):
    """(1 - b) p0 + b p1 [+ offset] in float64 with the bound of lerp_rn (1 - b, two products, the sum: one rounding each; the offset add
    one more)."""
    p0, p1, b = f64(p0), f64(p1), f64(b)
    a0, a1 = (1.0 - b) * p0, b * p1
    y = a0 + a1
    tol = U32 * (2 * a0.abs() + a1.abs() + y.abs())
    if offset is not None:
        y = y + f64(offset)
        tol = tol + U32 * y.abs()
    return y, tol


def slerp_cands(a, b, t) -> List[Cand]:
    """torch_utils.slerp of fp32 rows a, b [..., 4] at the kernel's fp32 blend t (broadcast to [..., 1]), float64, one candidate per
    branch outcome the fp32 kernel can reach (module docstring)."""
    a, b, t = f64(a), f64(b), f64(t)
    prod = a * b
    c = prod.sum(-1)
    dc = 5 * U32 * prod.abs().sum(-1)
    out: List[Cand] = []
    tt = t.expand(a.shape[:-1] + (1,))[..., 0]
    for sign in (1.0, -1.0):
        ok_sign = (c > -dc) if sign > 0 else (c < dc)                # the kernel flips b iff its c < 0
        cc = sign * c
        bb = sign * b
        s2 = 1.0 - cc * cc
        ds2 = 2 * cc.abs() * dc + dc * dc + U32
        s_lo = torch.sqrt(torch.clamp(s2 - ds2, min=0.0)) * (1 - U32)
        s_hi = torch.sqrt(torch.clamp(s2 + ds2, min=0.0)) * (1 + U32)
        must_one = cc > 1.0 + dc
        out.append((a, torch.zeros_like(a), ok_sign & (cc >= 1.0 - dc)))
        mid = 0.5 * a + 0.5 * bb
        out.append((mid, U32 * mid.abs(), ok_sign & ~must_one & (s_lo < SLERP_MID)))
        s_min = torch.clamp(s_lo, min=SLERP_MID * (1 - U32))
        h = torch.acos(torch.clamp(cc, -1.0, 1.0))
        s = torch.sqrt(torch.clamp(s2, min=0.0))
        e_h = _acos_err(torch.clamp(cc, -1.0, 1.0), dc)
        safe = torch.where(s > 0, s, torch.ones_like(s))
        ra = torch.where(s > 0, torch.sin((1 - tt) * h) / safe, 1 - tt)
        rb = torch.where(s > 0, torch.sin(tt * h) / safe, tt)
        eta = U32 / (2 * s_min * s_min) + U32                          # the fp32 c^2 (and 1 - c^2) rounding, through the root
        rel = 15 * U32 + eta                                           # arguments, sin polynomial, fdiv_fast, the product
        e_abs = 0.25 * (h + e_h) * (e_h + 4 * U32 * h) + 1e-9 / s_min  # the slope of the weights against h; polynomial truncation
        ta = (ra.abs() * rel + e_abs)[..., None] * a.abs()
        tb = (rb.abs() * rel + e_abs)[..., None] * bb.abs()
        y = ra[..., None] * a + rb[..., None] * bb
        tol = ta + tb + 2 * U32 * ((ra[..., None] * a).abs() + (rb[..., None] * bb).abs()) + U32 * y.abs()
        out.append((y, tol, ok_sign & ~must_one & (s_hi >= SLERP_MID)))
    return out


def expmap_cands(q, tq) -> List[Cand]:
    """quat_to_exp_map of q [..., 4] known to within tq (per component) of the kernel's input, float64: candidates for the s <= 1e-5 zero,
    the plain angle and the angle wrapped past pi (module docstring)."""
    w, v = q[..., 3], q[..., :3]
    dw, dv = tq[..., 3], tq[..., :3].amax(-1)
    s2 = 1.0 - w * w
    ds2 = 2 * w.abs() * dw + dw * dw + 2 * U32
    s = torch.sqrt(torch.clamp(s2, min=0.0))
    s_lo = torch.sqrt(torch.clamp(s2 - ds2, min=0.0)) * (1 - U32)
    s_hi = torch.sqrt(torch.clamp(s2 + ds2, min=0.0)) * (1 + U32)
    zero = torch.zeros_like(v)
    out: List[Cand] = [(zero, zero, s_lo <= EXP_EPS * (1 + U32))]
    live = s_hi > EXP_EPS * (1 - U32)
    s_min = torch.clamp(s_lo, min=EXP_EPS * (1 - U32))
    ang = 2.0 * torch.acos(torch.clamp(w, -1.0, 1.0))
    e_ang = 2 * _acos_err(torch.clamp(w, -1.0, 1.0), dw) + 4 * U32 * ang
    ds = ds2 / (2 * s_min) + U32 * s_hi
    safe = torch.where(s > 0, s, s_min)
    for wrapped in (False, True):
        a = ang - 2 * math.pi if wrapped else ang
        ea = e_ang + (abs(TWO_PI32 - 2 * math.pi) + U32 * a.abs() if wrapped else 0.0)
        ok = live & ((ang + e_ang >= math.pi) if wrapped else (ang - e_ang < PI32))
        e = (a / safe)[..., None] * v
        tol = ((v.norm(dim=-1) / s_min) * ea + a.abs() / s_min * dv)[..., None] + e.abs() * (ds / s_min + 5 * U32)[..., None]
        out.append((e, tol, ok))
    return out


def query_ref(tb, ids, times, blend, offset=None) -> Dict[str, object]:
    """get_motion_state on tables tb (dict of the float32 tables, any body count) at the kernel's fp32 blend: {"i0", "i1", "blend"}
    from oracle.pulse_oracle.frame_blend (exact), (ref, tol) for the lerped fields, candidates for the rotations and dof positions."""
    from oracle import pulse_oracle as po
    ids = ids.long()
    i0, i1, b_ref = po.frame_blend(times, tb["lengths"][ids], tb["num_frames"][ids], tb["dt"][ids])
    f0 = i0 + tb["length_starts"][ids]
    f1 = i1 + tb["length_starts"][ids]
    bb = blend[:, None, None]
    out: Dict[str, object] = {"i0": i0, "i1": i1, "blend": b_ref}
    out["rg_pos"] = lerp_ref(tb["gts"][f0], tb["gts"][f1], bb, None if offset is None else offset[:, None, :])
    out["body_vel"] = lerp_ref(tb["gvs"][f0], tb["gvs"][f1], bb)
    out["body_ang_vel"] = lerp_ref(tb["gavs"][f0], tb["gavs"][f1], bb)
    out["dof_vel"] = lerp_ref(tb["dvs"][f0].reshape(len(ids), -1), tb["dvs"][f1].reshape(len(ids), -1), blend[:, None])
    out["rb_rot"] = slerp_cands(tb["grs"][f0], tb["grs"][f1], bb)
    dof = []
    for q, t, ok in slerp_cands(tb["lrs"][f0][:, 1:], tb["lrs"][f1][:, 1:], bb):
        dof += [(e, te, ok & oe) for e, te, oe in expmap_cands(q, t)]
    out["dof_pos"] = dof
    if "motion_aa" in tb:
        out["motion_aa"] = tb["motion_aa"][f0]
    return out


def root_cands(cands: List[Cand]) -> List[Cand]:
    """The candidates of body 0 (root_rot from rb_rot's)."""
    return [(v[:, 0], t[:, 0], ok[:, 0]) for v, t, ok in cands]


def check_query(rep: Optional[Report], tag: str, got: Dict[str, torch.Tensor], ref: Dict[str, object], built=None,
                diagnostics: bool = True) -> None:
    """Every output of one query against query_ref: indices and blend exactly, lerps element-wise, rotations by branch."""
    if diagnostics:
        check_exact(rep, f"{tag} frame_idx0", got["frame_idx0"], ref["i0"])
        check_exact(rep, f"{tag} frame_idx1", got["frame_idx1"], ref["i1"])
        check_exact(rep, f"{tag} blend", got["blend"], ref["blend"])
    if "rg_pos" in got:
        for k in ("rg_pos", "body_vel", "body_ang_vel", "dof_vel"):
            check(rep, f"{tag} {k}", got[k], *ref[k])
        for k, body in (("root_pos", "rg_pos"), ("root_vel", "body_vel"), ("root_ang_vel", "body_ang_vel")):
            check(rep, f"{tag} {k}", got[k], ref[body][0][:, 0], ref[body][1][:, 0])
        rb_built = None if built is None else built[:, None]
        check_branches(rep, f"{tag} rb_rot (slerp)", got["rb_rot"], ref["rb_rot"], built=rb_built)
        check_branches(rep, f"{tag} root_rot (slerp)", got["root_rot"], root_cands(ref["rb_rot"]), built=built)
        n = got["dof_pos"].shape[0]
        check_branches(rep, f"{tag} dof_pos (slerp, exp map)", got["dof_pos"].reshape(n, -1, 3), ref["dof_pos"], built=rb_built)
        if "motion_aa" in got:
            check_exact(rep, f"{tag} motion_aa", got["motion_aa"], ref["motion_aa"])
    else:
        check(rep, f"{tag} root_pos", got["root_pos"], ref["rg_pos"][0][:, 0], ref["rg_pos"][1][:, 0])


# ------------------------------------------------------------------------------------------------------------------ test inputs
SMPL_PARENTS = [-1, 0, 1, 2, 3, 0, 5, 6, 7, 0, 9, 10, 11, 12, 11, 14, 15, 16, 17, 11, 19, 20, 21, 22]


def _aa_to_quat(aa):
    ang = aa.norm(dim=-1, keepdim=True)
    axis = aa / ang.clamp_min(1e-12)
    return torch.cat([axis * torch.sin(0.5 * ang), torch.cos(0.5 * ang)], -1)


def loader_clips(lengths, rates, seed: int, headings="mixed"):
    """On-disk-schema clips for the loader (float64 global rotations [T, 24, 4] and root translation [T, 3]): smooth rotations turning up to
    ~0.6 rad per frame, every third clip's quaternions stored with w < 0, every clip's scaled off unit length by up to 1e-3, every
    fourth clip's root rotation turning past pi within the clip.  headings "mixed": 0, pi, -pi, then uniform draws; None: no heading step.
    Returns (quat [F, 24, 4], trans [F, 3], frame_clip int32 [F], clip_start int64 [M + 1], fps float64 [M], headings float64 [M] or None,
    local_translation float32 [24, 3])."""
    g = torch.Generator().manual_seed(seed)
    M = len(lengths)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    quats, trans = [], []
    for c, (n, r) in enumerate(zip(lengths, rates)):
        speed = rn(1, 24, 3) * (2.0 + 10.0 * (c % 3)) / r             # rad per frame: slow, medium, fast clips
        aa = rn(1, 24, 3) + torch.cumsum(speed + 0.2 * speed.abs().amax() * rn(n, 24, 3), 0)
        if c % 4 == 1:
            aa[:, 0] = torch.linspace(0.0, 1.0, n, dtype=torch.float64)[:, None] * torch.tensor([0.0, 0.0, 4.0], dtype=torch.float64) \
                + torch.tensor([0.0, 0.0, 1.2], dtype=torch.float64)
        q = _aa_to_quat(aa)
        if c % 3 == 0:
            q = -q
        q = q * (1.0 + 1e-3 * (2 * torch.rand(n, 24, 1, generator=g, dtype=torch.float64) - 1))
        quats.append(q)
        trans.append(torch.cumsum(rn(n, 3) * 0.02, 0) + torch.tensor([0.0, 0.0, 0.9], dtype=torch.float64))
    nf = torch.tensor(lengths, dtype=torch.int64)
    clip_start = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(nf, 0)])
    frame_clip = torch.repeat_interleave(torch.arange(M, dtype=torch.int32), nf)
    if headings == "mixed":
        hd = (2 * torch.rand(M, generator=g, dtype=torch.float64) - 1) * math.pi
        hd[: min(3, M)] = torch.tensor([0.0, math.pi, -math.pi], dtype=torch.float64)[: min(3, M)]
    else:
        hd = None
    loc = (0.12 * torch.randn(24, 3, generator=g)).float()
    loc[0] = 0.0
    return torch.cat(quats), torch.cat(trans), frame_clip, clip_start, torch.tensor(rates, dtype=torch.float64), hd, loc
