"""The float64 AMP row of the 52-body SMPL-X humanoid (PULSE-X, env_pulsex_amp.yaml), with the element-wise bounds of the kernels'
fp32 operations: build_amp_observations_smpl with the SMPL-X dof_subset (the 49 joints 0..50 without L_Toe and R_Toe), key bodies
(7, 3, 36, 17) and the heading of remove_base_rot(root) (has_upright_start False).  466 floats, 465 without the root height:
[h | six(hinv q0) | R v0 | R w0 | 49 x six(dof) | 147 dof velocities | 4 x R(key - p0)].

The rotation, heading and exponential-map links and their bounds are tests/reset_fp64.py's (base_removed, heading_ref, yaw_qmul,
yaw_apply, six_ref, expmap_six_cands, primary); only the joint and key-body tables and the column layout are SMPL-X's."""
import math
from typing import Dict, Optional

import torch

from tests import motion_fp64 as mf
from tests import reset_fp64 as rf
from tests.fp64_ref import U32, Report, check, f64

BODIES, DOFS = 52, 153
KEPT_JOINTS = [j for j in range(BODIES - 1) if j not in (3, 7)]
KEY_BODIES = [7, 3, 36, 17]
J = len(KEPT_JOINTS)
AMP_OBS, AMP_OBS_NO_HEIGHT = 13 + 9 * J + 12, 12 + 9 * J + 12
AMP_COLS = {"h": (0, 1), "root": (1, 7), "vel": (7, 10), "ang": (10, 13), "dof_six": (13, 13 + 6 * J), "dof_vel": (13 + 6 * J, 13 + 9 * J),
            "key": (13 + 9 * J, AMP_OBS)}
DOF_SUBSET = [3 * j + c for j in KEPT_JOINTS for c in range(3)]


def amp_row_ref(p0, tp0, q0, tq0, v0, tv0, w0, tw0, dof, tdof, dvel, tdvel, key, tkey, upright: bool = False) -> Dict[str, object]:
    """rf.amp_row_ref in the SMPL-X layout: dof [n, 51, 3] with Euclidean bounds tdof [n, 51], dof velocities [n, 153], key-body
    positions [n, 4, 3] (bodies 7, 3, 36, 17).  Returns (ref, tol) per column group, "dof_six" candidates [n, 49, 6] and "ill"."""
    qb, tqb = rf.base_removed(q0, tq0, upright)
    hs, hc, dth, ill = rf.heading_ref(qb, tqb, True)
    rq, trq = rf.yaw_qmul(hs, hc, dth, qb, tqb)
    out: Dict[str, object] = {"h": (p0[:, 2:3], tp0[:, 2:3]), "root": rf.six_ref(rq, trq), "vel": rf.yaw_apply(hs, hc, dth, v0, tv0),
                              "ang": rf.yaw_apply(hs, hc, dth, w0, tw0), "ill": ill}
    kj = torch.tensor(KEPT_JOINTS, device=dof.device)
    out["dof_six"] = rf.expmap_six_cands(dof[:, kj], tdof[:, kj])
    vi = torch.tensor(DOF_SUBSET, device=dof.device)
    out["dof_vel"] = (dvel[:, vi], tdvel[:, vi])
    rel = key - p0[:, None, :]
    trel = tkey + tp0[:, None, :] + U32 * rel.abs()
    k, tk = rf.yaw_apply(hs[:, None], hc[:, None], dth[:, None], rel, trel)
    out["key"] = (k.reshape(len(p0), 12), tk.reshape(len(p0), 12))
    return out


def check_amp(rep: Optional[Report], tag: str, got: torch.Tensor, ref: Dict[str, object], built: Optional[torch.Tensor] = None) -> None:
    """rf.check_amp for SMPL-X rows of 466 or 465 floats."""
    width = got.shape[-1]
    skip = AMP_OBS - width
    n = got.shape[0]
    for name, (a, b) in AMP_COLS.items():
        if name == "h" and skip:
            continue
        g = got[:, a - skip:b - skip]
        if name == "dof_six":
            mf.check_branches(rep, f"{tag} amp dof six", g.reshape(n, J, 6), ref["dof_six"])
        else:
            r, t = ref[name]
            if name in ("root", "vel", "ang", "key"):
                t = torch.where(ref["ill"][:, None], torch.full_like(t, math.inf), t)
            check(rep, f"{tag} amp {name}", g, r, t)
    rf.limit_share(rep, f"{tag} amp heading", ref["ill"], built)


def state_amp_ref(body: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, upright: bool = False) -> Dict[str, object]:
    """amp_row_ref of a simulator state: body [n, >= 52, 13], dof_pos / dof_vel [n, 153], all exact fp32."""
    b = f64(body)
    z = lambda t: torch.zeros_like(t)
    kb = torch.tensor(KEY_BODIES, device=b.device)
    dof = f64(dof_pos).reshape(len(b), BODIES - 1, 3)
    return amp_row_ref(b[:, 0, 0:3], z(b[:, 0, 0:3]), b[:, 0, 3:7], z(b[:, 0, 3:7]), b[:, 0, 7:10], z(b[:, 0, 7:10]), b[:, 0, 10:13],
                       z(b[:, 0, 10:13]), dof, torch.zeros(dof.shape[:2], dtype=dof.dtype, device=dof.device), f64(dof_vel),
                       z(f64(dof_vel)), b[:, kb, 0:3], z(b[:, kb, 0:3]), upright)


def motion_amp_ref(q: Dict[str, object], upright: bool = False) -> Dict[str, object]:
    """amp_row_ref of the un-fixed motion (rf.motion_ref over the 52-body tables): the primary slerp / exp-map candidates."""
    pos, tpos = q["rg_pos"]
    vel, tvel = q["body_vel"]
    ang, tang = q["body_ang_vel"]
    rr, trr, amb_r = rf.primary(mf.root_cands(q["rb_rot"]))
    dof, tdof, amb_d = rf.primary(q["dof_pos"])
    dv, tdv = q["dof_vel"]
    kb = torch.tensor(KEY_BODIES, device=pos.device)
    ref = amp_row_ref(pos[:, 0], tpos[:, 0], rr, trr, vel[:, 0], tvel[:, 0], ang[:, 0], tang[:, 0], dof, tdof.norm(dim=-1), dv, tdv,
                      pos[:, kb], tpos[:, kb], upright)
    ref["ill"] = ref["ill"] | amb_r | amb_d.any(-1)
    return ref


def ref_values(ref: Dict[str, object], width: int) -> torch.Tensor:
    """The float64 row [n, width] of a reference: every group's value, the joints' primary rotation-feature candidate."""
    six, _, _ = rf.primary(ref["dof_six"])
    parts = [ref["root"][0], ref["vel"][0], ref["ang"][0], six.reshape(six.shape[0], -1), ref["dof_vel"][0], ref["key"][0]]
    if width == AMP_OBS:
        parts.insert(0, ref["h"][0])
    return torch.cat(parts, -1)
