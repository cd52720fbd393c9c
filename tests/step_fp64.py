"""Teacher-forced float64 references of the task step kernels (ztask_env.cuh: ztask_env<SmplReachLayout | SmplLayout |
SmplxLayout | SmplxTargetLayout>; terrain.cu: terrain_env; ztask_step.cu: reach_update_task_kernel; amp_obs.cu), each output with an element-wise
bound derived from the fp32 operations its kernel performs (the style of tests/fp64_ref.py and tests/reset_fp64.py, whose comparators,
heading and rotation references are reused).

Every reference is fed the fp32 inputs the kernel read (body states, contact forces, targets, prev_root_pos, trajectory vertices, the
height field) and recomputes each output in float64:

* heading: heading_half (the latent-task steps) and heading_quat_ref (atan2 + sincosf, the terrain task's height points and trajectory
  samples) both land within reset_fp64.heading_ref's angle bound dth -- the rotated x axis' roundings over its length 1 / |(rx, ry)|,
  plus 16 u32 for the half-angle / trigonometric step; every heading-frame output carries dth |v_xy|.  rx = ry = 0 exactly gives heading 0
  (the kernels' atan2(0, 0) branch) and is decided exactly; a heading whose axis is shorter than four times its bound is ill-conditioned
  and passes any rotation-dependent value, its share limited.
* self observation: [root height | (B - 1) local positions | B six-D rotations of yaw (x) q | B local velocities | B angular velocities],
  358 floats for SMPL (B = 24), 778 for SMPL-X (B = 52).  The SMPL-X steps take the heading of remove_base_rot(root); their task
  observation keeps the raw root's.  The two are separate links ("self ..." and "task ..."), so swapping them fails a named link.
* rewards: float64 with the bound of each fp32 operation (expf: 2 ulp); a reward that takes a branch on a rounded quantity (strike
  rot_err < 0.2 and dir_speed <= 0, terrain fuzzy err < 0.0025) has one candidate per branch the bound allows, and the share of rows
  with two is limited.  rot_err is also evaluated in fp32 in every order contraction can give it; when they all agree the decision is
  exact.
* decisions: contact |f| > 0.1, z < termination height, strike contacts > 50, progress > 1, progress >= max_len - 1 read fp32 inputs and
  are exact; terrain's force-sum norm > 50 and `far` are decided from rounded sums and may go either way within their bound.
* terrain: cell index trunc(x / h) clipped to [0, dim - 2]; a point within its bound of a cell edge may take either neighbour and its
  height must then equal that cell's min(h1, h2) vscale exactly.  The center height (a mean over the 3 x 3 center points) is checked
  against the interval its reachable cells give; those points are multiples of the cell size, so their edge share is limited by
  reset_fp64.EDGE_MAX as in the spawn reset.

The imitation step (im_step.cu: im_step_kernel, both the 934-float row and the tracked row) and the general task observation
(task_obs.cu) have their own references, im_step_ref and task_obs_ref:

* planner, exact: t_rew = motion_time_rn(prog), t_obs = motion_time_rn(prog + 1 - rec) (three fp32 roundings in the reference's order),
  the frame rows and blend of oracle.pulse_oracle.frame_blend (pinned to frame_blend_rn by tests/test_gpu_motion_fp64.py), the
  pass_time mask, progress_rw under PULSE_STEP_ADVANCE and the getup pull-back, fdones_out.  The blend is an exact operand of every
  later link, as in motion_fp64.query_ref.
* reference pose at t_rew and t_obs: query_ref on the tables plus global_offset -- lerps for position and velocities, slerp candidates
  for the rotations, slerp + exponential map candidates for ref_dof_pos (the aux records of the observation rows, joints 1..23).
* reward: the position / velocity / angular-velocity sums sum_j |r_j - x_j|^2 carry the lerp bound through the squares (2 |d| td + td^2),
  sq3's three roundings and the 24 roundings of the column sum; the mean's fp32 constant 1 / 72 (or 1 / 24) is off by at most u32
  relative and its product rounds once; k * e rounds once; expf is exp_neg's 2 ulp.  The rotation error is the angle of
  r.q (x) conj(q): 2 acos(w) wrapped past fp32(pi) as oracle.pulse_oracle.wrap_angle wraps it, with acos conditioned by
  motion_fp64._acos_err near w = +-1 and the s <= 1e-5 zero branch; w is known within r.q's slerp bound times |q|_1 plus the 8-product
  rounding (qmul8_err).  Every branch the bound allows (every allowed slerp candidate, then zero / plain / wrapped angle) gives a
  theta^2 interval; the body's term is that union, so the reward has one value and one bound, and rows where the slerp candidates
  differ (reset_fp64.primary) are counted, their share limited.  The power term is sum |tau qdot| (dof_power: 69 products, 2 adds
  per body thread and the 24-term column sum), zero at prog <= 3.  reward = sum w_i r_i + power within 5 u32 of its terms.
* reset: the per-body decision dist > termination_distances[j] is taken from an fp32 restatement in the kernel's pinned order
  (lerp_rn, the __fadd_rn offset, __fsub_rn, norm3_rn's two fused multiply-adds and the correctly rounded root), which makes it exact;
  the mean criterion sums those distances in body order and divides by popc(mask).  The float64 distance is a second link: the
  restatement must lie within its bound, and every row whose distances all lie outside their bound of the threshold must take the
  float64 decision; the share of rows that do not is limited.  prog > 1, early termination, cycle recovery and getup recovery are exact.
* observation at t_obs: self_obs_ref (upright), and the six pieces of the v6 task block, each its own link -- yaw_apply of r.p - p,
  r.v - v, r.w - w and r.p - p_root, six_ref of H^-1 (r.q (x) conj q) H (yaw_qmul, then yaw_qmul_right) and of H^-1 r.q.  Rows whose
  heading is ill-conditioned or whose r.q may take two slerp branches pass any rotation-dependent value; their share is limited.
* task_obs_ref: the same pieces from the fp32 ref_* arrays the kernel read (exact operands), the heading of body 0 through
  base_rot_removed(upright), in every version's layout (flat over (t, j) for 1, 2, 3; per sample for 6, 7, 8, 9), v8's R rv / R rw,
  v9's root-velocity pair from tracked body 0, and v2's dof difference, which is one fp32 rounding of the float64 difference: exact.
"""
import math
from typing import Dict, List, Optional

import numpy as np
import torch

from tests import motion_fp64 as mf
from tests import reset_fp64 as rf
from tests.fp64_ref import U32, BoundError, Report, check, check_exact, f32r, f64  # noqa: F401  (re-exported for the tests)

AMBIGUOUS_MAX = 1e-3
SPEED, STRIKE, REACH = 1, 2, 3
SMPL, SMPLX = 24, 52
NUM_DOF = 69
TRAJ_VERTS = 101
CONTACT_EPS, HARD_FORCE = f32r(0.1), 50.0
ROT_THRESH, FUZZY_THRESH = f32r(0.2), f32r(0.0025)


def self_obs_width(B: int) -> int:
    return 15 * B - 2


def r32(x: torch.Tensor) -> torch.Tensor:
    """x (float64) rounded to fp32 and back."""
    return x.float().double()


# ------------------------------------------------------------------------------------------------------------------ heading
def heading(q: torch.Tensor, upright: bool):
    """(hs, hc, dth, ill) of the heading of base_rot_removed(q) (q float64 [n, 4] of fp32 values): reset_fp64.heading_ref, with the
    exactly vertical x axis (rx = ry = 0 in exact arithmetic on an upright root, so also in fp32) decided as heading 0."""
    hs, hc, dth, ill = rf.heading_ref(q, torch.zeros_like(q), upright)
    if upright:
        x, y, z, w = q.unbind(-1)
        zero = ((2 * w * w - 1 + 2 * x * x) == 0) & ((2 * w * z + 2 * x * y) == 0)
        hs, hc = torch.where(zero, torch.zeros_like(hs), hs), torch.where(zero, torch.ones_like(hc), hc)
        dth, ill = torch.where(zero, torch.zeros_like(dth), dth), ill & ~zero
    return hs, hc, dth, ill


def yaw_apply(hs, hc, dth, v, tv):
    """reset_fp64.yaw_apply plus 16 u32 |v|: the kernels' (hs, hc) are unit only to a few u32 (rsqrtf, sqrtf and the divide of
    heading_half; atan2f / sincosf and the normalisation of heading_quat_ref), which scales every rotated vector, z included."""
    out, tol = rf.yaw_apply(hs, hc, dth, v, tv)
    return out, tol + 16 * U32 * v.norm(dim=-1, keepdim=True)


def _h(hd, extra: int = 0):
    hs, hc, dth, _ = hd
    sh = (slice(None),) + (None,) * extra
    return hs[sh], hc[sh], dth[sh]


# ------------------------------------------------------------------------------------------------------------------ self observation
def self_obs_ref(body: torch.Tensor, upright: bool, dz: Optional[torch.Tensor] = None, tdz: Optional[torch.Tensor] = None) -> Dict[str, object]:
    """The self observation of body [n, B, 13] (fp32 values, float64 or float32) in the heading of base_rot_removed(root, upright).
    dz [n] / tdz [n]: a height subtracted from every body's z first (the terrain's center height) and its bound.  Returns
    {link: (ref, tol)} over the layout's column groups and "ill"."""
    b = f64(body)
    n, B = b.shape[0], b.shape[1]
    p, q, v, w = b[..., 0:3].clone(), b[..., 3:7], b[..., 7:10], b[..., 10:13]
    tp = torch.zeros_like(p)
    if dz is not None:
        p[..., 2] = p[..., 2] - dz[:, None]
        tp[..., 2] = tdz[:, None] + U32 * p[..., 2].abs()
    hd = heading(q[:, 0], upright)
    hs, hc, dth = _h(hd, 1)
    rel = p[:, 1:] - p[:, 0:1]
    trel = tp[:, 1:] + tp[:, 0:1] + U32 * rel.abs()
    pos, tpos = yaw_apply(hs, hc, dth, rel, trel)
    rq, trq = rf.yaw_qmul(hs, hc, dth, q, torch.zeros_like(q))
    six, tsix = rf.six_ref(rq, trq)
    vel, tvel = yaw_apply(hs, hc, dth, v, torch.zeros_like(v))
    ang, tang = yaw_apply(hs, hc, dth, w, torch.zeros_like(w))
    fl = lambda t: t.reshape(n, -1)
    return {"root h": (p[:, 0, 2:3], tp[:, 0, 2:3]), "body pos": (fl(pos), fl(tpos)), "body six": (fl(six), fl(tsix)),
            "body vel": (fl(vel), fl(tvel)), "body ang": (fl(ang), fl(tang)), "ill": hd[3]}


def self_cols(B: int) -> Dict[str, tuple]:
    return {"root h": (0, 1), "body pos": (1, 3 * B - 2), "body six": (3 * B - 2, 9 * B - 2), "body vel": (9 * B - 2, 12 * B - 2),
            "body ang": (12 * B - 2, 15 * B - 2)}


def loose(t: torch.Tensor, ill: torch.Tensor) -> torch.Tensor:
    return torch.where(ill.reshape(ill.shape + (1,) * (t.dim() - 1)), torch.full_like(t, math.inf), t)


def check_self(rep: Optional[Report], tag: str, obs: torch.Tensor, ref: Dict[str, object], built: Optional[torch.Tensor] = None) -> None:
    B = ref["body six"][0].shape[1] // 6
    for name, (a, b) in self_cols(B).items():
        r, t = ref[name]
        check(rep, f"{tag} self {name}", obs[:, a:b], r, t if name == "root h" else loose(t, ref["ill"]))
    rf.limit_share(rep, f"{tag} self heading", ref["ill"], built)


# ------------------------------------------------------------------------------------------------------------------ the latent tasks
def dof_power(dof_force, dof_vel, adds: int = 8):
    """sum |f v| over the 69 dofs and its bound: the products (one rounding each), then `adds` roundings along the deepest chain of
    the kernel's sum -- 3 lane-local adds and 5 shuffle levels in the latent-task steps; 2 adds per body thread and the 24-term
    column sum in the imitation step."""
    t = (f64(dof_force)[:, :NUM_DOF] * f64(dof_vel)[:, :NUM_DOF]).abs()
    s = t.sum(-1)
    return s, (adds + 2) * U32 * s


def _root_vel(root, prev, dt):
    d = root[:, :2] - f64(prev)[:, :2]
    v = d / f32r(dt)
    return v, 2 * U32 * v.abs()


def exp_neg(a, ta):
    """expf(-a) for a >= 0 known within ta, and its bound (expf: 2 ulp; below fp32's smallest normal number the result may be a
    subnormal or 0)."""
    e = torch.exp(-a)
    return e, e * torch.expm1(ta) + 5 * U32 * e + 2.0 ** -126


def rot_err_orders(tq: torch.Tensor) -> torch.Tensor:
    """2 w^2 - 1 + 2 z^2 of fp32 quaternions [n, 4] in fp32 in each of the four orders FMA contraction can give it: [n, 4] float64."""
    z, w = f64(tq[:, 2]), f64(tq[:, 3])
    fma = lambda a, b, c: r32(a * b + c)           # a * b is exact in float64 for fp32 a, b
    ww, zz = r32(r32(2 * w) * w), r32(r32(2 * z) * z)
    s1, s2 = r32(ww - 1), fma(2 * w, w, torch.full_like(w, -1.0))
    return torch.stack([r32(s1 + zz), r32(s2 + zz), fma(2 * z, z, s1), fma(2 * z, z, s2)], -1)


def ztask_ref(kind: int, B: int, inp: Dict[str, torch.Tensor], obs_only: bool = False) -> Dict[str, object]:
    """One latent-task step (ztask_env in the layout of B and kind) on inputs `inp` (CPU tensors):
      body [n, B, 13], progress [n], and as the kind needs: contact [n, B, 3] (or None), term_h [B], contact_mask, strike_mask (ints),
      early (bool), max_len, prev [n, 3], dt, tar_speed [n], dof_force / dof_vel [n, 69] (or None), power_c, tar_pos [n, 3], reach_id,
      target [n, 13], tar_contact [n, 3].
    Returns {"self": self_obs_ref, "task": {link: (ref, tol)}, "task ill", and unless obs_only: "reward" candidates, "raw1" (ref, tol),
    "reset" / "terminate" exact int64, "rew_amb" rows}."""
    upright = B == SMPL
    b = f64(inp["body"])
    n = b.shape[0]
    root, rq = b[:, 0, 0:3], b[:, 0, 3:7]
    out: Dict[str, object] = {"self": self_obs_ref(b, upright)}
    hd = heading(rq, True)                    # the task observation: the raw root's heading
    hs, hc, dth = _h(hd)
    out["task ill"] = hd[3]
    task: Dict[str, tuple] = {}
    if kind == SPEED:
        e = torch.zeros(n, 3, dtype=torch.float64)
        e[:, 0] = 1.0
        d, td = yaw_apply(hs, hc, dth, e, torch.zeros_like(e))
        task["speed dir"] = (d[:, :2], td[:, :2])
        ts = f64(inp["tar_speed"])[:, None]
        task["speed target"] = (ts, torch.zeros_like(ts))
    elif kind == REACH:
        rel = f64(inp["tar_pos"]) - root
        task["reach target"] = yaw_apply(hs, hc, dth, rel, U32 * rel.abs())
    else:
        ts = f64(inp["target"])
        rel = torch.stack([ts[:, 0] - root[:, 0], ts[:, 1] - root[:, 1], ts[:, 2]], 1)
        trel = torch.stack([U32 * rel[:, 0].abs(), U32 * rel[:, 1].abs(), torch.zeros_like(rel[:, 2])], 1)
        task["strike pos"] = yaw_apply(hs, hc, dth, rel, trel)
        tq = ts[:, 3:7]
        task["strike six"] = rf.six_ref(*rf.yaw_qmul(hs, hc, dth, tq, torch.zeros_like(tq)))
        task["strike vel"] = yaw_apply(hs, hc, dth, ts[:, 7:10], torch.zeros_like(ts[:, 7:10]))
        task["strike ang"] = yaw_apply(hs, hc, dth, ts[:, 10:13], torch.zeros_like(ts[:, 10:13]))
    out["task"] = task
    if obs_only:
        return out

    # ---- reset: every decision reads fp32 inputs, exact
    prog = inp["progress"].long().cpu()
    early = bool(inp["early"])
    cm, sm = int(inp["contact_mask"]), int(inp.get("strike_mask", 0))
    bits = torch.tensor([(cm >> j) & 1 for j in range(B)], dtype=torch.bool)
    contact = torch.zeros(n, dtype=torch.bool)
    height = torch.zeros(n, dtype=torch.bool)
    if early:
        if inp.get("contact") is not None:
            f = inp["contact"].float()[:, :B].abs()
            contact = ((f > CONTACT_EPS).any(-1) & ~bits[None]).any(-1)
        height = ((inp["body"].float()[:, :B, 2] < inp["term_h"].float()[None, :B]) & ~bits[None]).any(-1)
    failed = contact & height
    if kind == STRIKE and early:
        sbits = torch.tensor([((cm | sm) >> j) & 1 for j in range(B)], dtype=torch.bool)
        hard = torch.zeros(n, dtype=torch.bool)
        if inp.get("contact") is not None:
            hard = ((inp["contact"].float()[:, :B].abs() > HARD_FORCE).any(-1) & ~sbits[None]).any(-1)
        tc = inp["tar_contact"].float().abs()
        failed = failed | ((tc[:, 0] > HARD_FORCE) | (tc[:, 1] > HARD_FORCE)) & hard
    term = (early & failed & (prog > 1)).long()
    out["terminate"] = term
    out["reset"] = torch.where(prog >= int(inp["max_len"]) - 1, torch.ones_like(term), term)

    # ---- reward
    ones = torch.ones(n, dtype=torch.bool)
    if kind == SPEED:
        v, tv = _root_vel(root, inp["prev"], inp["dt"])
        ts = f64(inp["tar_speed"])
        err = ts - v[:, 0]
        terr = tv[:, 0] + U32 * err.abs()
        vy, tvy = v[:, 1], tv[:, 1]
        a = 0.25 * (err * err + 0.1 * vy * vy)
        ta = 0.25 * (2 * err.abs() * terr + terr * terr + 0.1 * (2 * vy.abs() * tvy + tvy * tvy)) + 5 * U32 * a
        rew, trew = exp_neg(a, ta)
        out["raw0"] = (rew[:, None], trew[:, None])
        pw, tpw = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
        if inp.get("dof_force") is not None:
            c = f32r(inp["power_c"])
            s, ts_ = dof_power(inp["dof_force"], inp["dof_vel"])
            live = prog > 3
            pw = torch.where(live, -c * s, pw)
            tpw = torch.where(live, c * ts_ + U32 * c * s, tpw)
        out["raw1"] = (pw[:, None], tpw[:, None])
        tot = rew + pw
        out["reward"] = [(tot[:, None], (trew + tpw + U32 * tot.abs())[:, None], ones)]
    elif kind == REACH:
        d = f64(inp["tar_pos"]) - b[:, int(inp["reach_id"]), 0:3]
        td = U32 * d.abs()
        s = (d * d).sum(-1)
        a = 4 * s
        ta = 4 * ((2 * d.abs() * td + td * td).sum(-1) + 4 * U32 * s)
        rew, trew = exp_neg(a, ta)
        out["reward"] = [(rew[:, None], trew[:, None], ones)]
    else:
        ts = f64(inp["target"])
        tq = ts[:, 3:7]
        z, w = tq[:, 2], tq[:, 3]
        rot = 2 * w * w - 1 + 2 * z * z
        trot = 4 * U32 * (2 * w * w + 1 + 2 * z * z)
        o = rot_err_orders(inp["target"][:, 3:7])
        same = (o == o[:, :1]).all(-1)
        lt_sure = torch.where(same, o[:, 0] < ROT_THRESH, rot + trot < ROT_THRESH)
        ge_sure = torch.where(same, o[:, 0] >= ROT_THRESH, rot - trot >= ROT_THRESH)
        rot_r = torch.clamp(1 - rot, min=0.0)
        trr = trot + U32
        v, tv = _root_vel(root, inp["prev"], inp["dt"])
        dxy = ts[:, 0:2] - root[:, 0:2]
        tdxy = U32 * dxy.abs()
        dn = dxy.norm(dim=-1)
        zero_dir = dn == 0                                  # target directly above the root: normalize's 1e-12 floor gives (0, 0)
        dn_s = torch.where(zero_dir, torch.ones_like(dn), dn)
        u = torch.where(zero_dir[:, None], torch.zeros_like(dxy), dxy / dn_s[:, None])
        tdn = (dxy.abs() * tdxy).sum(-1) / dn_s + 3 * U32 * dn
        tu = torch.where(zero_dir[:, None], torch.zeros_like(u), tdxy / dn_s[:, None] + u.abs() * (tdn / dn_s)[:, None] + U32 * u.abs())
        ds = (u * v).sum(-1)
        tds = (u.abs() * tv + tu * v.abs() + tu * tv).sum(-1) + 3 * U32 * (u * v).abs().sum(-1)
        zero_ds = zero_dir | (v == 0).all(-1)               # prev_root_pos == root, or no direction: dir_speed is exactly 0
        tds = torch.where(zero_ds, torch.zeros_like(tds), tds)
        ds = torch.where(zero_ds, torch.zeros_like(ds), ds)
        pos_sure = ~zero_ds & (ds - tds > 0)
        npos_sure = zero_ds | (ds + tds <= 0)
        verr = torch.clamp(1 - ds, min=0.0)
        tverr = tds + U32 * verr
        vel_r, tvel = exp_neg(4 * verr * verr, 4 * (2 * verr * tverr + tverr * tverr) + 3 * U32 * 4 * verr * verr)
        cands = [(torch.ones(n, 1, dtype=torch.float64), torch.zeros(n, 1, dtype=torch.float64), ~ge_sure)]
        for vr, tvr, ok in ((vel_r, tvel, ~npos_sure), (torch.zeros_like(vel_r), torch.zeros_like(tvel), ~pos_sure)):
            r = 0.6 * rot_r + 0.4 * vr
            cands.append((r[:, None], (0.6 * trr + 0.4 * tvr + 3 * U32 * r.abs())[:, None], ~lt_sure & ok))
        out["reward"] = cands
        out["rot_decided"] = lt_sure | ge_sure
        out["dir_decided"] = pos_sure | npos_sure
    return out


def task_cols(kind: int, B: int) -> Dict[str, tuple]:
    s = self_obs_width(B)
    if kind == SPEED:
        return {"speed dir": (s, s + 2), "speed target": (s + 2, s + 3)}
    if kind == REACH:
        return {"reach target": (s, s + 3)}
    return {"strike pos": (s, s + 3), "strike six": (s + 3, s + 9), "strike vel": (s + 9, s + 12), "strike ang": (s + 12, s + 15)}


def check_obs(rep: Optional[Report], tag: str, kind: int, B: int, obs: torch.Tensor, ref: Dict[str, object],
              built: Optional[torch.Tensor] = None) -> None:
    """The observation rows [n, >= width] against ztask_ref: the self observation and the task observation, link by link."""
    check_self(rep, tag, obs[:, :self_obs_width(B)], ref["self"], built)
    for name, (a, b) in task_cols(kind, B).items():
        r, t = ref["task"][name]
        check(rep, f"{tag} task {name}", obs[:, a:b], r, t if name == "speed target" else loose(t, ref["task ill"]))
    rf.limit_share(rep, f"{tag} task heading", ref["task ill"], built)


def check_step(rep: Optional[Report], tag: str, kind: int, B: int, got: Dict[str, torch.Tensor], ref: Dict[str, object],
               built: Optional[torch.Tensor] = None) -> None:
    """A step's outputs (CPU tensors: obs [n, >= width], rew [n], reset / terminate int64 [n], raw [n, 1 or 2] or None) against
    ztask_ref."""
    check_obs(rep, tag, kind, B, got["obs"], ref, built)
    check_exact(rep, f"{tag} terminate", got["terminate"], ref["terminate"])
    check_exact(rep, f"{tag} reset", got["reset"], ref["reset"])
    if kind == SPEED and got.get("raw") is not None:
        raw = got["raw"]
        check(rep, f"{tag} reward raw speed", raw[:, 0:1], *ref["raw0"])
        if raw.shape[1] > 1 and got.get("power", False):
            check(rep, f"{tag} reward raw power", raw[:, 1:2], *ref["raw1"])
            check_exact(rep, f"{tag} reward = raw speed + raw power", got["rew"], (raw[:, 0] + raw[:, 1]))
        else:
            check_exact(rep, f"{tag} reward = raw speed", got["rew"], raw[:, 0])
    mf.check_branches(rep, f"{tag} reward", got["rew"].reshape(-1, 1), ref["reward"], built=built)


# ------------------------------------------------------------------------------------------------------------------ small entry points
def reach_update_ref(progress, change, tar, rand, steps, dist_max: float, h_min: float, h_max: float) -> Dict[str, tuple]:
    """pulse_reach_update_task: the due envs (progress >= change) take reset_fp64.task_ref's target and change steps, the others keep
    theirs bit for bit.  Returns {"due", "target": (ref, tol), "change"}."""
    due = progress.long() >= change.long()
    t = rf.task_ref("reach", rand, steps, progress, dist_max, h_min, h_max, 0.0, 1.0)
    v, tol = t["target"]
    v = torch.where(due[:, None], v, f64(tar))
    tol = torch.where(due[:, None], tol, torch.zeros_like(tol))
    return {"due": due, "target": (v, tol), "change": torch.where(due, t["change_steps"], change.long())}


def amp_obs_ref(body, dof_pos, dof_vel) -> Dict[str, object]:
    """pulse_amp_obs's new row: build_amp_observations_smpl of the simulator state (root heading of the root itself)."""
    return rf.state_amp_ref(body[:, :SMPL], dof_pos, dof_vel, True)


# ------------------------------------------------------------------------------------------------------------------ terrain
def traj_ref(verts: torch.Tensor, t: torch.Tensor, traj_dt: float):
    """TrajGenerator.calc_pos of waypoints verts [n, V, 3] at fp32 times t [n, K]: phase = clip(t / (V traj_dt), 0, 1) -- V, not V - 1 --
    then the lerp between waypoints floor / ceil(phase (V - 1)).  float64 [n, K, 3] with the bound: the phase and segment position are
    known within 3 u32 (the quotient, the fp32 duration, the product), the path is continuous in it (so a segment boundary is not a
    branch), and the lerp rounds four times."""
    v = f64(verts)
    n, V = v.shape[0], v.shape[1]
    tt = f64(t)
    phase = torch.clamp(tt / (V * traj_dt), 0.0, 1.0)
    seg = phase * (V - 1)
    tseg = 3 * U32 * seg
    i0 = torch.clamp(torch.floor(seg).long(), 0, V - 2)
    b = seg - i0.double()
    g = lambda idx: torch.gather(v, 1, idx.reshape(n, -1, 1).expand(-1, -1, 3))
    p0, p1 = g(i0), g(i0 + 1)
    pos = p0 + b[..., None] * (p1 - p0)
    # slope: the larger of the two segments that meet at a boundary within the segment bound
    ilo = torch.clamp(i0 - 1, 0, V - 2)
    ihi = torch.clamp(i0 + 1, 0, V - 2)
    slope = torch.maximum((p1 - p0).abs(), torch.maximum((g(ilo + 1) - g(ilo)).abs(), (g(ihi + 1) - g(ihi)).abs()))
    tol = slope * tseg[..., None] + 4 * U32 * (p0.abs() + p1.abs())
    return pos, tol


def cells(hf: torch.Tensor, hscale: float, vscale: float, x: torch.Tensor, y: torch.Tensor, tx: torch.Tensor, ty: torch.Tensor):
    """The heights sample_height may return for a world point known within (tx, ty) of (x, y) (float64 of any shape): the cells of the
    interval's two ends in each axis (trunc of the fp32 quotient, clipped to [0, dim - 2]), min(h1, h2) * vscale in fp32.  Returns
    (heights [..., 4] float64 of the candidate cells, edge: the point's cell is not decided)."""
    R, Cc = hf.shape
    h32 = f32r(hscale)
    q = lambda c, top: (c / h32).float().trunc().long().clamp(0, top)   # fp32 quotient through float64 (innocuous double rounding)
    xa, xb = q(x - tx, R - 2), q(x + tx, R - 2)
    ya, yb = q(y - ty, Cc - 2), q(y + ty, Cc - 2)
    hfi = hf.long()
    hts = []
    for px in (xa, xb):
        for py in (ya, yb):
            hts.append((torch.minimum(hfi[px, py], hfi[px + 1, py + 1]).float() * torch.tensor(vscale, dtype=torch.float32)).double())
    return torch.stack(hts, -1), (xa != xb) | (ya != yb)


def points_world(q: torch.Tensor, tq_angle: torch.Tensor, pts: torch.Tensor, origin: torch.Tensor):
    """quat_apply(yaw q, offset) + origin for yaw quaternions q [n, 4] (float64, exact up to the angle bound tq_angle [n]) and offsets pts
    [P, 3]: world xy [n, P] each, and their bounds (the angle bound times |offset|, quat_apply_rn's 12 u32 |offset|, the add)."""
    z, w = q[:, 2:3], q[:, 3:4]
    c, s = w * w - z * z, 2 * w * z
    px, py = pts[None, :, 0], pts[None, :, 1]
    rx, ry = c * px - s * py, s * px + c * py
    r = pts[:, :2].norm(dim=-1)[None, :]
    dr = r * (tq_angle[:, None] + 12 * U32)
    x, y = rx + origin[:, 0:1], ry + origin[:, 1:2]
    return x, y, dr + U32 * x.abs(), dr + U32 * y.abs()


def yaw_only_ref(q: torch.Tensor, upright: bool):
    """yaw_only(base_rot_removed(q)) float64 [n, 4] and its angle bound: 2 (tz + tw) / |(z, w)| plus the roundings; ill where |(z, w)| is
    within four times the component bound."""
    qb, tqb = rf.base_removed(q, torch.zeros_like(q), upright)
    nz = torch.sqrt(qb[:, 2] ** 2 + qb[:, 3] ** 2)
    e = tqb[:, 2] + tqb[:, 3] + 2 * U32 * nz
    ill = e * 4 >= nz
    ns = torch.where(ill, torch.ones_like(nz), nz)
    out = torch.stack([torch.zeros_like(nz), torch.zeros_like(nz), qb[:, 2] / ns, qb[:, 3] / ns], -1)
    return out, torch.where(ill, torch.full_like(nz, 2 * math.pi), 2 * e / ns + 8 * U32), ill


def center_ref(hf, hscale, vscale, q, pos, pts, upright: bool):
    """The mean center height around (pos [n, 3], q [n, 4]) over pts [P, 3]: (mid, half-width + rounding bound, rows with a point
    within its bound of a cell edge, rows whose yaw is ill-conditioned -- their bound is infinite)."""
    p = f64(pts)
    P = p.shape[0]
    if hf is None:
        z = torch.zeros(q.shape[0], dtype=torch.float64)
        return z, z.clone(), torch.zeros(q.shape[0], dtype=torch.bool), torch.zeros(q.shape[0], dtype=torch.bool)
    qy, dphi, ill = yaw_only_ref(f64(q), upright)
    x, y, tx, ty = points_world(qy, dphi, p, f64(pos))
    hts, edge = cells(hf, hscale, vscale, x, y, tx, ty)
    lo, hi = hts.amin(-1).sum(-1) / P, hts.amax(-1).sum(-1) / P
    tol = 0.5 * (hi - lo) + 6 * U32 * hts.abs().amax(-1).sum(-1) / P
    tol = torch.where(ill, torch.full_like(tol, math.inf), tol)
    return 0.5 * (lo + hi), tol, edge.any(-1), ill


def terrain_ref(inp: Dict[str, object], flags: int) -> Dict[str, object]:
    """terrain_env on inputs (CPU): body [n, 24, 13] (rigid bodies), root [n, 13] (actor root), progress [n] (as the kernel saw it),
    contact [n, 24, 3], contact_mask, early, no_collision, fuzzy, power_reward, upright, use_center_height, num_traj_samples,
    height_points [P, 3], center_points [Pc, 3], head_id, dt, traj_dt, sample_dt, fail_dist, power_c, verts [n, 101, 3], hf int16
    [R, C] or None, hscale, vscale, dof_force / dof_vel [n, 69] or None, max_len."""
    REW, RST, OBS = 1, 2, 4
    b = f64(inp["body"])
    n = b.shape[0]
    a_root = f64(inp["root"])
    prog = inp["progress"].long()
    t_now = prog.float() * torch.tensor(inp["dt"], dtype=torch.float32)       # __fmul_rn(__ll2float_rn(prog), dt)
    tar, ttar = traj_ref(inp["verts"], t_now[:, None], inp["traj_dt"])
    tar, ttar = tar[:, 0], ttar[:, 0]
    out: Dict[str, object] = {}
    ones = torch.ones(n, dtype=torch.bool)
    if flags & REW:
        d = tar[:, :2] - a_root[:, :2]
        td = ttar[:, :2] + U32 * d.abs()
        err = (d * d).sum(-1)
        terr = (2 * d.abs() * td + td * td).sum(-1) + 2 * U32 * err
        loc, tloc = exp_neg(2 * err, 2 * terr + U32 * 2 * err)
        power, tpow = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
        if inp.get("dof_force") is not None:
            c = f32r(inp["power_c"])
            s, ts_ = dof_power(inp["dof_force"], inp["dof_vel"])
            power, tpow = -c * s, c * ts_ + U32 * c * s
        one, zero = torch.ones_like(loc), torch.zeros_like(loc)
        if inp["fuzzy"]:
            near_ok = err - terr < FUZZY_THRESH
            far_ok = err + terr >= FUZZY_THRESH
            out["loc"] = [(one[:, None], zero[:, None], near_ok), (loc[:, None], tloc[:, None], far_ok)]
        else:
            out["loc"] = [(loc[:, None], tloc[:, None], ones)]
        out["power"] = (power[:, None], tpow[:, None])
        if inp["power_reward"]:
            out["reward"] = [(v + power[:, None], t + tpow[:, None] + U32 * (v + power[:, None]).abs(), ok) for v, t, ok in out["loc"]]
        else:
            out["reward"] = out["loc"]
    if flags & RST:
        early = bool(inp["early"])
        cm = int(inp["contact_mask"])
        bits = torch.tensor([(cm >> j) & 1 for j in range(SMPL)], dtype=torch.bool)
        f = f64(inp["contact"])[:, :SMPL] * (~bits)[None, :, None]
        s = f.sum(1)
        ts_ = SMPL * U32 * f.abs().sum(1)
        nrm = s.norm(dim=-1)
        tn = (s.abs() * ts_).sum(-1) / torch.where(nrm > 0, nrm, torch.ones_like(nrm)) + (ts_ * ts_).sum(-1).sqrt() + 3 * U32 * nrm
        # a row whose every partial sum, square and the root are fp32 numbers is computed exactly in any order
        part = torch.cumsum(f, 1)
        sq = s * s
        exact = ((r32(part) == part).all(1).all(-1) & (r32(sq) == sq).all(-1) & (r32(sq[:, :2].sum(-1)) == sq[:, :2].sum(-1))
                 & (r32(sq.sum(-1)) == sq.sum(-1)) & (r32(nrm) == nrm))
        tn = torch.where(exact, torch.zeros_like(tn), tn)
        fall_hi = (nrm + tn > HARD_FORCE) & (prog > 1)
        fall_lo = (nrm - tn > HARD_FORCE) & (prog > 1)
        d = tar[:, :2] - b[:, 0, :2]                        # the rigid-body root
        td = ttar[:, :2] + U32 * d.abs()
        d2 = (d * d).sum(-1)
        td2 = (2 * d.abs() * td + td * td).sum(-1) + 2 * U32 * d2
        fd = f32r(f32r(inp["fail_dist"]) * f32r(inp["fail_dist"]))
        far_hi, far_lo = d2 + td2 > fd, d2 - td2 > fd
        live = early and not inp["no_collision"]
        t_hi = (fall_hi | far_hi) & live
        t_lo = (fall_lo | far_lo) & live
        out["term_lo"], out["term_hi"] = t_lo.long(), t_hi.long()
        out["reset_floor"] = prog >= int(inp["max_len"]) - 1
    if flags & OBS:
        upright = bool(inp["upright"])
        hf = inp.get("hf")
        c_self, tc_self, edge_self, ill_self = center_ref(hf, inp["hscale"], inp["vscale"], b[:, 0, 3:7], b[:, 0, 0:3], inp["center_points"],
                                                          upright)
        out["self"] = self_obs_ref(b, upright, dz=c_self, tdz=tc_self)
        out["self"]["ill"] = out["self"]["ill"] | ill_self
        out["self edge"] = edge_self
        # trajectory samples at t_now + k sample_dt (both fp32 roundings exact), in the actor root's heading_quat_ref frame
        K = int(inp["num_traj_samples"])
        k = torch.arange(K, dtype=torch.float32)
        tk = t_now[:, None] + k[None, :] * torch.tensor(inp["sample_dt"], dtype=torch.float32)
        tp, ttp = traj_ref(inp["verts"], tk, inp["traj_dt"])
        rel = tp - a_root[:, None, 0:3]
        trel = ttp + U32 * rel.abs()
        hd = heading(a_root[:, 3:7], True) if upright else rf.heading_ref(a_root[:, 3:7], torch.zeros_like(a_root[:, 3:7]), False)
        hs, hc, dth = _h(hd, 1)
        lt, tlt = yaw_apply(hs, hc, dth, rel, trel)
        out["traj"] = (lt[..., :2].reshape(n, 2 * K), loose(tlt[..., :2].reshape(n, 2 * K), hd[3]))
        out["traj ill"] = hd[3]
        # height map at the head pose relative to ref_h, clipped to +-3 m and scaled by 5
        if inp["use_center_height"]:
            ref_h, tref, edge_ref, ill_ref = center_ref(hf, inp["hscale"], inp["vscale"], a_root[:, 3:7], a_root[:, 0:3], inp["center_points"],
                                                        upright)
        else:
            ref_h, tref = a_root[:, 2], torch.zeros(n, dtype=torch.float64)
            edge_ref, ill_ref = torch.zeros(n, dtype=torch.bool), torch.zeros(n, dtype=torch.bool)
        pts = f64(inp["height_points"])
        P = pts.shape[0]
        if hf is None:
            m = torch.zeros(n, P, 1, dtype=torch.float64)
            edge = torch.zeros(n, P, dtype=torch.bool)
            hill = torch.zeros(n, dtype=torch.bool)
        else:
            head = b[:, int(inp["head_id"])]
            hh = heading(head[:, 3:7], True) if upright else rf.heading_ref(head[:, 3:7], torch.zeros_like(head[:, 3:7]), False)
            hq = torch.stack([torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), hh[0], hh[1]], -1)
            x, y, tx, ty = points_world(hq, hh[2], pts, head[:, 0:3])
            m, edge = cells(hf, inp["hscale"], inp["vscale"], x, y, tx, ty)
            hill = hh[3]
        val = torch.clamp(ref_h[:, None, None] - m, -3.0, 3.0) * 5.0
        tol = 5 * (tref[:, None, None] + U32 * (ref_h[:, None, None] - m).abs()) + U32 * val.abs()
        tol = torch.where(hill[:, None, None], torch.full_like(tol, math.inf), tol)
        # candidate 0 is the cell of the interval's lower ends; the others are allowed only for a point on a cell edge
        cands = [(val[..., c:c + 1], tol[..., c:c + 1], torch.ones(n, P, dtype=torch.bool) if c == 0 else edge) for c in range(m.shape[-1])]
        out["heights"] = cands
        out["num_height_points"] = P
        out["heights edge"] = edge | hill[:, None]                 # per point
        out["ref edge"] = edge_ref | ill_ref
    return out


def check_terrain(rep: Optional[Report], tag: str, flags: int, got: Dict[str, torch.Tensor], ref: Dict[str, object], K: int,
                  built: Optional[torch.Tensor] = None) -> None:
    """terrain_env's outputs against terrain_ref, for the flag subset `flags`.  got: obs [n, >= width], rew [n], raw [n, 2] or None,
    reset / terminate [n]."""
    if flags & 1:
        mf.check_branches(rep, f"{tag} reward", got["rew"].reshape(-1, 1), ref["reward"], built=built)
        if got.get("raw") is not None:
            raw = got["raw"]
            mf.check_branches(rep, f"{tag} reward raw location", raw[:, 0:1], ref["loc"], built=built)
            check(rep, f"{tag} reward raw power", raw[:, 1:2], *ref["power"])
            want = raw[:, 0] + raw[:, 1] if got.get("power_reward") else raw[:, 0]
            check_exact(rep, f"{tag} reward = raw columns", got["rew"], want)
    if flags & 2:
        term, lo, hi = got["terminate"].long(), ref["term_lo"], ref["term_hi"]
        wrong = (term != lo) & (term != hi)
        rep is not None and rep.add(f"{tag} terminate (exact outside the bound)", float(wrong.any()))
        if wrong.any():
            k = int(torch.nonzero(wrong)[0])
            raise BoundError(f"{tag} terminate: {int(wrong.sum())} rows outside the decided value, first env {k}: got {int(term[k])}, "
                             f"allowed {int(lo[k])} / {int(hi[k])}")
        rf.limit_share(rep, f"{tag} terminate", lo != hi, built)
        check_exact(rep, f"{tag} reset", got["reset"], torch.where(ref["reset_floor"], torch.ones_like(term), term))
    if flags & 4:
        obs = got["obs"]
        self_ = ref["self"]
        check_self(rep, tag, obs[:, :358], self_, built)
        rf.limit_share(rep, f"{tag} self center height cell edge", ref["self edge"], built, amb_max=rf.EDGE_MAX)
        check(rep, f"{tag} traj samples", obs[:, 358:358 + 2 * K], *ref["traj"])
        rf.limit_share(rep, f"{tag} traj heading", ref["traj ill"], built)
        hobs = obs[:, 358 + 2 * K:358 + 2 * K + ref["num_height_points"]]
        mf.check_branches(rep, f"{tag} heights", hobs[..., None], ref["heights"], built=None if built is None else built[:, None])
        rf.limit_share(rep, f"{tag} heights cell edge", ref["heights edge"], None if built is None else built[:, None])
        rf.limit_share(rep, f"{tag} heights center height cell edge", ref["ref edge"], built, amb_max=rf.EDGE_MAX)


# ------------------------------------------------------------------------------------------------------------------ imitation step
IM_SELF, IM_TASK = 358, 576
REW, RST, OBS, ADVANCE = 1, 2, 4, 8
IM_PIECES = (("dp", 3), ("drot", 6), ("dv", 3), ("dw", 3), ("lp", 3), ("lrot", 6))     # the v6 task block, block-major over the bodies
EXP_EPS = 1e-5


def motion_time32(prog: torch.Tensor, dt: float, start: torch.Tensor, off: torch.Tensor) -> torch.Tensor:
    """motion_time_rn: fp32(progress) * dt + start + offset, three fp32 roundings (torch rounds each CPU float32 operation)."""
    return (prog.long().float() * torch.tensor(dt, dtype=torch.float32) + start.float()) + off.float()


def fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fmaf of fp32 tensors, rounded once: a * b is exact in float64; the float64 sum's own rounding error e is recovered exactly
    (two-sum) and decides the one case where rounding twice differs from rounding once -- a float64 sum exactly halfway between two
    fp32 numbers."""
    p = a.double() * b.double()
    cc = c.double()
    s = p + cc
    bb = s - p
    e = (p - (s - bb)) + (cc - bb)
    r = s.float()
    other = torch.nextafter(r, torch.where(s > r.double(), torch.full_like(r, math.inf), torch.full_like(r, -math.inf)))
    half = (s == 0.5 * (r.double() + other.double())) & (e != 0) & (s != r.double())
    up = torch.where(e > 0, torch.maximum(r, other), torch.minimum(r, other))
    return torch.where(half, up, r)


def lerp_rn32(p0: torch.Tensor, p1: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """lerp_rn: ((1 - b) p0) + (b p1), every operation rounded on its own."""
    return (1.0 - b) * p0 + b * p1


def reset_dist32(p0, p1, b, goff, pos) -> torch.Tensor:
    """The kernel's termination distance in its pinned fp32 order: r.p = lerp_rn + __fadd_rn offset, __fsub_rn, norm3_rn =
    sqrt(fma(z, z, fma(y, y, x x))).  p0 / p1 [n, B, 3] the frame rows, b [n, 1, 1] the blend, goff [n, 1, 3], pos [n, B, 3]."""
    rp = lerp_rn32(p0.float(), p1.float(), b.float()) + goff.float()
    d = pos.float() - rp
    x, y, z = d.unbind(-1)
    return torch.sqrt(fma32(z, z, fma32(y, y, x * x)))


def yaw_qmul_right(hs, hc, dth, q, tq):
    """qmul(q, (0, 0, hs, hc)) -- the right multiply by the forward heading that closes H^-1 (x) q (x) H -- in float64 with its bound,
    as reset_fp64.yaw_qmul: pairwise mixing, |q| dth / 2, the 8-product rounding."""
    h = torch.stack([torch.zeros_like(hs), torch.zeros_like(hs), hs, hc], -1).expand(q.shape)
    out = mf.qmul(q, h)
    pair = torch.stack([tq[..., 0] + tq[..., 1], tq[..., 0] + tq[..., 1], tq[..., 2] + tq[..., 3], tq[..., 2] + tq[..., 3]], -1)
    return out, pair + (0.5 * q.norm(dim=-1) * dth.expand(q.shape[:-1]))[..., None] + mf.qmul8_err(q, h)


def rel_rot(rq, trq, q):
    """r.q (x) conj(q) of fp32 simulator quaternions q in float64, with its bound: r.q's bound times |q|_1 per component, and the
    8-product rounding."""
    qc = mf.qconj(q)
    return mf.qmul(rq, qc), (trq.amax(-1) * q.abs().sum(-1))[..., None] + mf.qmul8_err(rq, qc)


def angle_cands(w: torch.Tensor, dw: torch.Tensor) -> List[mf.Cand]:
    """quat_angle (quat_to_angle_axis's angle) of a quaternion whose w is known within dw: candidates [..., 1] for the s <= 1e-5 zero,
    2 acos(w), and 2 acos(w) - 2 pi past fp32(pi), with motion_fp64.expmap_cands' conditioning (acosf 2 ulp, the wrap's fp32 2 pi)."""
    s2 = 1.0 - w * w
    ds2 = 2 * w.abs() * dw + dw * dw + 2 * U32
    s_lo = torch.sqrt(torch.clamp(s2 - ds2, min=0.0)) * (1 - U32)
    s_hi = torch.sqrt(torch.clamp(s2 + ds2, min=0.0)) * (1 + U32)
    live = s_hi > EXP_EPS * (1 - U32)
    wc = torch.clamp(w, -1.0, 1.0)
    ang = 2.0 * torch.acos(wc)
    e_ang = 2 * mf._acos_err(wc, dw) + 4 * U32 * ang
    zero = torch.zeros_like(w)[..., None]
    out: List[mf.Cand] = [(zero, zero, s_lo <= EXP_EPS * (1 + U32))]
    out.append((ang[..., None], e_ang[..., None], live & (ang - e_ang < mf.PI32)))
    wa = ang - 2 * math.pi
    out.append((wa[..., None], (e_ang + abs(mf.TWO_PI32 - 2 * math.pi) + U32 * wa.abs())[..., None], live & (ang + e_ang >= math.pi)))
    return out


def _sq_interval(cands: List[mf.Cand]):
    """The union over the allowed candidates of [(|a| - t)^2, (|a| + t)^2] (one more rounding for the fp32 square): (mid, half-width)."""
    lo = hi = None
    for v, t, ok in cands:
        a, e = v[..., 0].abs(), t[..., 0]
        l, h = torch.clamp(a - e, min=0.0) ** 2 * (1 - U32), (a + e) ** 2 * (1 + U32)
        l = torch.where(ok, l, torch.full_like(l, math.inf))
        h = torch.where(ok, h, torch.full_like(h, -math.inf))
        lo, hi = (l, h) if lo is None else (torch.minimum(lo, l), torch.maximum(hi, h))
    return 0.5 * (lo + hi), 0.5 * (hi - lo)


def _sum_sq(d, td):
    """sum over bodies of |d_j|^2 for fp32 differences d [n, B, 3] known within td: the squares (2 |d| td + td^2), sq3's three
    roundings, and the B roundings of the column's running sum."""
    sq = (d * d).sum(-1)
    S = sq.sum(-1)
    return S, ((2 * d.abs() * td + td * td).sum(-1) + 3 * U32 * sq).sum(-1) + d.shape[1] * U32 * S


def _mean_exp(S, tS, cnt: int, k: float):
    """expf(-k (S * fp32(1 / cnt))) against exp(-k S / cnt): the constant's rounding (u32 relative), the two products, exp_neg."""
    c, kk = f32r(1.0 / cnt), f32r(k)
    e = S / cnt
    te = tS * c + abs(c - 1.0 / cnt) * S + U32 * e
    a = kk * e
    return exp_neg(a, kk * te + U32 * a)


def im_pose(tb, ids, t32, goff):
    """query_ref at fp32 times t32 with oracle.pulse_oracle.frame_blend's blend as the exact operand, plus the global frame rows.
    A clip of one frame has length 0, and at time 0 the phase is 0 / 0: frame_blend_rn's fmaxf / fminf take the NaN to phase 0, where
    the float reference would index with NaN.  Such a clip's rows are 0 and 0 whatever its length, so it is queried with length 1."""
    from oracle import pulse_oracle as po
    tb = {k: v for k, v in tb.items() if k != "motion_aa"}
    tb["lengths"] = torch.where(tb["lengths"] == 0, torch.ones_like(tb["lengths"]), tb["lengths"])
    i0, i1, b = po.frame_blend(t32, tb["lengths"][ids], tb["num_frames"][ids], tb["dt"][ids])
    q = mf.query_ref(tb, ids, t32, b, goff)
    q["f0"], q["f1"] = i0 + tb["length_starts"][ids], i1 + tb["length_starts"][ids]
    return q


def im_step_ref(tb, inp: Dict[str, object], cfg) -> Dict[str, object]:
    """One pulse_im_step launch on the envs of inp (CPU): body [n, 24, 13], progress (as read) [n], motion_ids, start, offset [n],
    goff [n, 3], cycle [n] int32 or None, recovery [n] int32 or None, dof_force / dof_vel [n, 69] or None, term [24] fp32, mask (int),
    flags (PULSE_STEP_* bits, ADVANCE included).  cfg: an ImConfig (dt, reward_specs, power_coefficient, enable_early_termination,
    cycle_motion, max_episode_length, use_mean_reset).  tb: the float32 tables as a dict.
    Returns the exact planner outputs ("pass_time", "progress", "reset", "terminate", "fdones"), the reward links, the fp64 reset links,
    the observation pieces ("self", "task" {piece: (ref [n, 24, w], tol)}, "obs ill"), the side buffers and the four-row count."""
    flags = int(inp["flags"])
    do_rew, do_reset, do_obs = bool(flags & REW), bool(flags & RST), bool(flags & OBS)
    need_t = do_rew or do_reset
    body = inp["body"].float()[:, :24]
    b64 = f64(body)
    n = body.shape[0]
    ids = inp["motion_ids"].long()
    prog = inp["progress"].long() + (1 if flags & ADVANCE else 0)
    rec = torch.zeros(n, dtype=torch.bool)
    if do_reset and inp.get("recovery") is not None:
        rec = inp["recovery"].int() > 0
    start, off, goff = inp["start"].float(), inp["offset"].float(), inp["goff"].float()
    t_rew = motion_time32(prog, cfg.dt, start, off)
    t_obs = motion_time32(prog + 1 - rec.long(), cfg.dt, start, off)
    mlen = tb["lengths"][ids].float()
    out: Dict[str, object] = {"t_rew": t_rew, "t_obs": t_obs}
    pos, rot, vel, ang = b64[..., 0:3], b64[..., 3:7], b64[..., 7:10], b64[..., 10:13]
    amb_rows = torch.zeros(n, dtype=torch.bool)
    if need_t:
        q1 = im_pose(tb, ids, t_rew, goff)
        out["pass_time"] = (t_rew >= mlen).to(torch.uint8)
    if do_obs:
        q2 = im_pose(tb, ids, t_obs, goff)
    if need_t and do_obs:
        rows = torch.stack([q1["f0"], q1["f1"], q2["f0"], q2["f1"]], 1)
        srt = rows.sort(1).values
        out["four"] = int(((srt[:, 1:] != srt[:, :-1]).sum(1) == 3).sum())
    # progress counter: the planner's advance, the recovering env's pull-back
    progress = inp["progress"].long().clone()
    if flags & ADVANCE:
        progress = torch.where(rec, progress, prog)
    progress = torch.where(rec, prog - 1, progress)
    out["progress"] = progress

    if do_rew:
        spec = cfg.reward_specs
        rp, trp = q1["rg_pos"]
        d = rp - pos
        S, tS = _sum_sq(d, trp + U32 * d.abs())
        r_pos = _mean_exp(S, tS, 72, spec["k_pos"])
        raw = [r_pos]
        for key, x in (("body_vel", vel), ("body_ang_vel", ang)):
            v, tv = q1[key]
            d = v - x
            raw.append(_mean_exp(*_sum_sq(d, tv + U32 * d.abs()), 72, spec["k_vel" if key == "body_vel" else "k_ang_vel"]))
        # rotation: the union of theta^2 over every allowed slerp candidate and angle branch
        mids, halves = [], []
        th_c: List[mf.Cand] = []
        for v, t, ok in q1["rb_rot"]:
            dq, tdq = rel_rot(v, t, rot)
            th_c += [(a, ta, ok & oa) for a, ta, oa in angle_cands(dq[..., 3], tdq[..., 3])]
        mid, half = _sq_interval(th_c)
        Sr = mid.sum(-1)
        r_rot = _mean_exp(Sr, half.sum(-1) + 24 * U32 * (mid + half).sum(-1), 24, spec["k_rot"])
        _, _, slerp_amb = rf.primary(q1["rb_rot"])
        out["rot amb"] = slerp_amb.any(-1)
        amb_rows |= out["rot amb"]
        raw = [raw[0], r_rot, raw[1], raw[2]]
        w = [f32r(spec[k]) for k in ("w_pos", "w_rot", "w_vel", "w_ang_vel")]
        tot = sum(wi * r for wi, (r, _) in zip(w, raw))
        ttot = sum(wi * t for wi, (_, t) in zip(w, raw)) + 5 * U32 * sum(wi * r.abs() for wi, (r, _) in zip(w, raw))
        power = None
        if inp.get("dof_force") is not None:
            c = f32r(cfg.power_coefficient)
            s, ts_ = dof_power(inp["dof_force"], inp["dof_vel"], adds=2 + 23)
            live = prog > 3
            pw = torch.where(live, -c * s, torch.zeros_like(s))
            tpw = torch.where(live, c * ts_ + U32 * c * s, torch.zeros_like(s))
            power = (pw, tpw)
            tot = tot + pw
            ttot = ttot + tpw + 5 * U32 * pw.abs()
        out["raw"] = raw + ([power] if power is not None else [])
        out["reward"] = (tot, ttot + U32 * tot.abs())

    if do_reset:
        mask = int(inp["mask"])
        bits = torch.tensor([(mask >> j) & 1 for j in range(24)], dtype=torch.bool)
        term = inp["term"].float()
        fr = tb["gts"]
        d32 = reset_dist32(fr[q1["f0"]], fr[q1["f1"]], q1["blend"][:, None, None], goff[:, None, :], body[..., 0:3])
        rp, trp = q1["rg_pos"]
        dd = pos - rp
        d64 = dd.norm(dim=-1)
        td64 = (trp + U32 * dd.abs()).norm(dim=-1) + 3 * U32 * d64
        out["dist"] = (d32, d64, td64)
        cnt = bin(mask & 0xFFFFFF).count("1")
        first = (mask & -mask).bit_length() - 1
        if cfg.use_mean_reset:
            m32 = torch.zeros(n, dtype=torch.float32)
            for j in range(24):
                m32 = m32 + torch.where(bits[j], d32[:, j], torch.zeros_like(m32))
            fell = m32 / torch.tensor(float(cnt), dtype=torch.float32) > term[first]
            md = (d64 * bits).sum(-1) / cnt
            tmd = ((td64 * bits).sum(-1) + 24 * U32 * (d64 * bits).sum(-1)) / cnt + U32 * md
            t0 = float(term[first])
            fell_lo, fell_hi = md - tmd > t0, md + tmd > t0
        else:
            fell = ((d32 > term[None]) & bits[None]).any(-1)
            fell_lo = ((d64 - td64 > f64(term)[None]) & bits[None]).any(-1)
            fell_hi = ((d64 + td64 > f64(term)[None]) & bits[None]).any(-1)
        pass_time = (prog >= int(cfg.max_episode_length) - 1) if cfg.cycle_motion else (t_rew >= mlen)
        cyc = inp["cycle"].int() if inp.get("cycle") is not None else torch.zeros(n, dtype=torch.int32)
        hold = (~pass_time & (cyc > 0)) | rec
        live = (prog > 1) & bool(cfg.enable_early_termination) & ~hold

        def decide(f):
            t = (f & live).long()
            return torch.where(hold, torch.zeros_like(t), torch.where(pass_time, torch.ones_like(t), t)), t

        out["reset"], out["terminate"] = decide(fell)
        out["term_lo"], out["term_hi"] = decide(fell_lo)[1], decide(fell_hi)[1]
        out["fdones"] = out["reset"].float()

    if do_obs:
        out["self"] = self_obs_ref(body, True)
        hd = heading(rot[:, 0], True)
        hs, hc, dth = _h(hd, 1)
        rp, trp = q2["rg_pos"]
        rv, trv = q2["body_vel"]
        rw, trw = q2["body_ang_vel"]
        rq, trq, amb2 = rf.primary(q2["rb_rot"])
        rel = lambda a, ta, b_: (a - b_, ta + U32 * (a - b_).abs())
        task = {"dp": yaw_apply(hs, hc, dth, *rel(rp, trp, pos)),
                "dv": yaw_apply(hs, hc, dth, *rel(rv, trv, vel)),
                "dw": yaw_apply(hs, hc, dth, *rel(rw, trw, ang)),
                "lp": yaw_apply(hs, hc, dth, *rel(rp, trp, pos[:, 0:1].expand_as(pos)))}
        dq, tdq = rel_rot(rq, trq, rot)
        task["drot"] = rf.six_ref(*yaw_qmul_right(hs, hc, dth, *rf.yaw_qmul(hs, hc, dth, dq, tdq)))
        task["lrot"] = rf.six_ref(*rf.yaw_qmul(hs, hc, dth, rq, trq))
        out["task"] = task
        out["obs ill"] = hd[3] | amb2.any(-1)
        amb_rows |= out["obs ill"]
        out["ref_body_pos"], out["ref_body_vel"] = q2["rg_pos"], q2["body_vel"]
        out["ref_body_rot"], out["ref_dof_pos"] = q2["rb_rot"], q2["dof_pos"]
    out["amb"] = amb_rows
    return out


def im_task_block(ref: Dict[str, object], track: Optional[tuple] = None):
    """The task block of the row as (ref, tol) [n, width] plus {piece: (first column, last column)}: the 576-float v6 block, or the
    tracked block of track = (version, ids), whose columns humanoid_im.track_columns selects from the v6 block."""
    from pulse_b200.humanoid_im import TRACK_BLOCKS, track_columns
    n = ref["task"]["dp"][0].shape[0]
    full = torch.cat([ref["task"][k][0].reshape(n, -1) for k, _ in IM_PIECES], 1)
    tol = torch.cat([loose(ref["task"][k][1], ref["obs ill"]).reshape(n, -1) for k, _ in IM_PIECES], 1)
    widths = dict(IM_PIECES)
    if track is None:
        cols, names, K = torch.arange(IM_TASK), [k for k, _ in IM_PIECES], 24
    else:
        version, tids = track
        cols, K = track_columns(version, tids), len(tids)
        at = {24 * sum(wd for _, wd in IM_PIECES[:i]): k for i, (k, _) in enumerate(IM_PIECES)}     # v6 offset -> piece
        names = [at[off] for off, _ in TRACK_BLOCKS[version]]
    spans, c0 = {}, 0
    for k in names:
        spans[k] = (c0, c0 + widths[k] * K)
        c0 += widths[k] * K
    return full[:, cols], tol[:, cols], spans


def check_im_step(rep: Optional[Report], tag: str, got: Dict[str, torch.Tensor], ref: Dict[str, object], flags: int,
                  track: Optional[tuple] = None, built: Optional[torch.Tensor] = None) -> None:
    """A step's outputs on the envs of the reference (CPU tensors: obs [n, >= width], self_obs [n, 358] or None, rew [n], raw
    [n, >= 4] or None, reset / terminate int64, pass_time uint8, progress int64, fdones float or None, ref_body_* / ref_dof_pos or
    None) against im_step_ref, link by link."""
    if flags & (REW | RST):
        check_exact(rep, f"{tag} pass_time", got["pass_time"], ref["pass_time"])
    if got.get("progress") is not None:
        check_exact(rep, f"{tag} progress", got["progress"], ref["progress"])
    if flags & REW:
        names = ("pos", "rot", "vel", "ang vel", "power")
        if got.get("raw") is not None:
            for c, (r, t) in enumerate(ref["raw"]):
                check(rep, f"{tag} reward raw {names[c]}", got["raw"][:, c], r, t)
        check(rep, f"{tag} reward", got["rew"], *ref["reward"])
        rf.limit_share(rep, f"{tag} reward rot slerp branch", ref["rot amb"], built)
    if flags & RST:
        d32, d64, td64 = ref["dist"]
        check(rep, f"{tag} reset distance (fp32 restatement)", d32, d64, td64)
        term = got["terminate"].long()
        wrong = (term != ref["term_lo"]) & (term != ref["term_hi"])
        rep is not None and rep.add(f"{tag} terminate (fp64 decided)", float(wrong.any()))
        if wrong.any():
            k = int(torch.nonzero(wrong)[0])
            raise BoundError(f"{tag} terminate (fp64 decided): {int(wrong.sum())} rows contradict the float64 distances, first env {k}: "
                             f"got {int(term[k])}, allowed {int(ref['term_lo'][k])} / {int(ref['term_hi'][k])}")
        rf.limit_share(rep, f"{tag} terminate within the distance bound", ref["term_lo"] != ref["term_hi"], built)
        check_exact(rep, f"{tag} terminate", term, ref["terminate"])
        check_exact(rep, f"{tag} reset", got["reset"], ref["reset"])
        if got.get("fdones") is not None:
            check_exact(rep, f"{tag} fdones", got["fdones"], ref["fdones"])
    if flags & OBS:
        obs = got["obs"]
        check_self(rep, tag, obs[:, :IM_SELF], ref["self"], built)
        if got.get("self_obs") is not None:
            check_exact(rep, f"{tag} self_obs_buf = obs[:, :358]", got["self_obs"], obs[:, :IM_SELF])
        r, t, spans = im_task_block(ref, track)
        for k, (a, b) in spans.items():
            check(rep, f"{tag} task {k}", obs[:, IM_SELF + a:IM_SELF + b], r[:, a:b], t[:, a:b])
        rf.limit_share(rep, f"{tag} task heading / slerp branch", ref["obs ill"], built)
        if got.get("ref_body_pos") is not None:
            check(rep, f"{tag} ref body pos", got["ref_body_pos"], *ref["ref_body_pos"])
            check(rep, f"{tag} ref body vel", got["ref_body_vel"], *ref["ref_body_vel"])
            bb = None if built is None else built[:, None]
            mf.check_branches(rep, f"{tag} ref body rot", got["ref_body_rot"], ref["ref_body_rot"], built=bb)
            mf.check_branches(rep, f"{tag} ref dof pos", got["ref_dof_pos"].reshape(-1, 23, 3), ref["ref_dof_pos"], built=bb)


# ------------------------------------------------------------------------------------------------------------------ task observation
# (piece, width, columns per unit of J, constant) in each version's layout; "flat" layouts index items it = t J + j over all samples,
# "per_t" layouts repeat the pieces per sample with a stride of the listed total
TASK_LAYOUT = {
    1: ("flat", [("dp", 3, 0, 0), ("drot", 6, 3, 0), ("dv", 3, 9, 0), ("dw", 3, 12, 0)]),
    2: ("flat", [("dp", 3, 0, 0), ("drot", 6, 3, 0), ("dv", 3, 9, 0), ("dw", 3, 12, 0)]),
    3: ("flat", [("dp", 3, 0, 0), ("drot", 6, 3, 0)]),
    6: ("per_t", [("dp", 3, 0, 0), ("drot", 6, 3, 0), ("dv", 3, 9, 0), ("dw", 3, 12, 0), ("lp", 3, 15, 0), ("lrot", 6, 18, 0)]),
    7: ("per_t", [("dp", 3, 0, 0), ("dv", 3, 3, 0), ("lp", 3, 6, 0)]),
    8: ("per_t", [("dp", 3, 0, 0), ("drot", 6, 3, 0), ("dv", 3, 9, 0), ("dw", 3, 12, 0), ("lp", 3, 15, 0), ("lrot", 6, 18, 0),
                  ("lv", 3, 24, 0), ("lw", 3, 27, 0)]),
    9: ("per_t", [("dp", 3, 0, 0), ("drot", 6, 3, 0), ("lp", 3, 9, 6), ("lrot", 6, 12, 6)]),
}


def task_obs_size(version: int, J: int, T: int) -> int:
    return {1: 15 * T * J, 2: 15 * J + 3 * (J - 1), 3: 9 * T * J, 6: 24 * T * J, 7: 9 * T * J, 8: 30 * J, 9: T * (18 * J + 6)}[version]


def task_obs_ref(version: int, T: int, track_ids, upright: bool, body, ref_pos, ref_rot, ref_vel, ref_ang, dof_pos=None,
                 ref_dof=None) -> Dict[str, object]:
    """pulse_im_task_obs on the fp32 arrays it read: body [n, 24, 13], ref_* [n T, 24, .] (row e T + t), dof_pos / ref_dof [n, 69].
    Returns {"links": [(name, columns [k], ref [n, k], tol [n, k])], "exact": [(name, columns, ref)], "ill": rows, "size"}."""
    b = f64(body)[:, :24]
    n = b.shape[0]
    ids = torch.as_tensor(list(track_ids), dtype=torch.long)
    J = len(ids)
    hd = heading(b[:, 0, 3:7], upright)
    hs, hc, dth = _h(hd, 2)
    g = lambda x, w: f64(x).reshape(n, T, 24, w)[:, :, ids]
    rp, rq, rv, rw = g(ref_pos, 3), g(ref_rot, 4), g(ref_vel, 3), g(ref_ang, 3)
    bt = b[:, ids][:, None]
    p, q, v, w = (bt[..., a:c].expand(n, T, J, c - a) for a, c in ((0, 3), (3, 7), (7, 10), (10, 13)))
    p_root = b[:, 0, 0:3][:, None, None].expand_as(p)
    diff = lambda a, c: yaw_apply(hs, hc, dth, a - c, U32 * (a - c).abs())
    pieces = {"dp": diff(rp, p), "dv": diff(rv, v), "dw": diff(rw, w), "lp": diff(rp, p_root),
              "lv": yaw_apply(hs, hc, dth, rv, torch.zeros_like(rv)), "lw": yaw_apply(hs, hc, dth, rw, torch.zeros_like(rw))}
    if version != 7:
        dq, tdq = rel_rot(rq, torch.zeros_like(rq), q)
        pieces["drot"] = rf.six_ref(*yaw_qmul_right(hs, hc, dth, *rf.yaw_qmul(hs, hc, dth, dq, tdq)))
        pieces["lrot"] = rf.six_ref(*rf.yaw_qmul(hs, hc, dth, rq, torch.zeros_like(rq)))
    kind, plist = TASK_LAYOUT[version]
    stride = {6: 24 * J, 7: 9 * J, 8: 30 * J, 9: 18 * J + 6}.get(version, 0)
    tt = torch.arange(T)[:, None, None]
    jj = torch.arange(J)[None, :, None]
    links = []
    for name, wd, cj, c0 in plist:
        cc = torch.arange(wd)[None, None, :]
        if kind == "flat":
            cols = cj * T * J + wd * (tt * J + jj) + cc
        else:
            cols = tt * stride + cj * J + c0 + wd * jj + cc
        r, t = pieces[name]
        links.append((name, cols.reshape(-1), r.reshape(n, -1), loose(t, hd[3]).reshape(n, -1)))
    if version == 9:                                    # root = tracked body 0: its velocity pair once per sample
        for name, key, c0 in (("root dv", "dv", 9 * J), ("root dw", "dw", 9 * J + 3)):
            r, t = pieces[key]
            cols = torch.arange(T)[:, None] * stride + c0 + torch.arange(3)[None, :]
            links.append((name, cols.reshape(-1), r[:, :, 0].reshape(n, -1), loose(t[:, :, 0], hd[3]).reshape(n, -1)))
    exact = []
    if version == 2:
        d0 = (3 * (ids[1:] - 1))[:, None] + torch.arange(3)[None, :]
        want = r32(f64(ref_dof)[:, d0.reshape(-1)] - f64(dof_pos)[:, d0.reshape(-1)])
        exact.append(("dof", 15 * J + torch.arange(3 * (J - 1)), want))
    return {"links": links, "exact": exact, "ill": hd[3], "size": task_obs_size(version, J, T)}


def check_task_obs(rep: Optional[Report], tag: str, obs: torch.Tensor, ref: Dict[str, object], built: Optional[torch.Tensor] = None) -> None:
    """pulse_im_task_obs rows [n, >= size] against task_obs_ref, one link per piece."""
    for name, cols, r, t in ref["links"]:
        check(rep, f"{tag} {name}", obs[:, cols], r, t)
    for name, cols, want in ref["exact"]:
        check_exact(rep, f"{tag} {name}", obs[:, cols], want)
    rf.limit_share(rep, f"{tag} heading", ref["ill"], built)
