"""Float64 reference of the evaluation metrics, frame by frame, with a deterministic bound on the fp32 kernel's deviation.

Every function takes the fp32 positions the kernel reads ([F, 24, 3] per frame: F frames, e.g. one per env of one step), evaluates the
definition in float64 and returns the value with a bound on |kernel - value|.  The definitions are those of `smpl_sim`'s
compute_metrics_lite as `oracle/eval_oracle.py` restates them (global / root-relative MPJPE, VideoPose3D `p_mpjpe`, the finite
differences of compute_error_vel / compute_error_accel); the bounds follow the fp32 operations of `csrc/eval_metrics.cu`:

* A subtraction of two fp32 values rounds once, relative to its result: |fl(a - b) - (a - b)| <= u32 |a - b|.  The positions the kernel
  reads are fp32 and the reference starts from those same values, so root-relative coordinates of a pose 10^3 m from the origin cost
  u32 |p_j - p_0|, not u32 |p_j|; the large-translation frame class of the GPU test holds the kernel to exactly that.
* A per-body norm sqrt(x^2 + y^2 + z^2) adds 3 u32 |v|.  The mean over the 24 bodies is a 5-level shuffle butterfly (5 u32 of the sum of
  the non-negative terms) times fl(1/24) (2 u32): 10 u32 of the value on top of the per-body errors.
* Procrustes (Horn's form, as the kernel computes it): the centred sets X (target) and Y (prediction), S[a][b] = sum_j Y_a X_b, the 4x4
  symmetric N(S) with ||N||_F = 2 ||S||_F, its largest eigenpair by cyclic Jacobi, scale = lambda / |Y|^2, R(q) applied to Y.
  With M = sum_j |Y_j| |X_j| the error of the computed N is at most E = 2 dS + 8 u32 M + C_JACOBI u32 ||N||_2, where dS bounds the
  error of S from the rounded coordinates and C_JACOBI covers the backward error of the Jacobi rotations (rsqrtf, a few roundings
  per rotation, six rotations per sweep over the sweeps that do not vanish).  Then
      |d lambda| <= E,   sin(angle(q, v1)) <= E / (gap - E)   (Davis-Kahan, gap = lambda1 - lambda2 of N in float64),
      ||R(q) - R(v1)||_2 <= 2 sin(angle),
  and the aligned residual s R Y_j - X_j of body j moves by at most s |Y_j| (ds / s + dR) plus the rounding of the coordinates.
  The value is a mean of distances, not the least-squares objective, so the rotation error enters at first order.
* Near-tied top eigenvalues (relative gap (lambda1 - lambda2) / lambda1 < TIE_GAP, or gap < 4 E): the eigenvector is not determined by
  N to fp32 accuracy, and the kernel may return any unit vector of span(v1, v2) (lambda3 is always separated: lambda1 - lambda3 >=
  2 sigma_1 of S).  The least-squares objective is flat on that span but the mean distance need not be (a mirror image of a pose whose
  two smaller principal moments are equal), so the bound is the range of the value over q(phi) = cos(phi) v1 + sin(phi) v2, phi on a
  grid of TIE_GRID points over [0, pi), widened by the grid's Lipschitz slack (|dR/dphi| = 2, so the value moves by at most
  2 s mean|Y| per radian), by the scale's spread (lambda anywhere in [lambda2 - E, lambda1 + E]) and by the rounding bound.  For
  collinear sets the range is empty (rotations about the common line move no body) and only the slack remains.  `pa_mpjpe` returns
  the mask of these frames and the report counts them.

All bounds are first order in u32; the second-order terms are below 1e-6 of them at the magnitudes used here.
"""
import math
from typing import Dict, List, Optional, Sequence

import numpy as np

U32 = 2.0 ** -24
U64 = 2.0 ** -53
J = 24
C_JACOBI = 64.0
TIE_GAP = 1e-4
TIE_GRID = 512
METRICS = ("mpjpe_g", "mpjpe_l", "mpjpe_pa", "vel_dist", "accel_dist")     # the columns of the kernel's sums[N, 5]


def _f64(a) -> np.ndarray:
    a = np.asarray(a)
    if a.dtype != np.float32:
        raise TypeError("the reference is evaluated on the fp32 positions the kernel reads")
    return a.astype(np.float64)


def _norm(v: np.ndarray) -> np.ndarray:
    return np.sqrt((v * v).sum(-1))


def _mean_norm(v: np.ndarray, e: np.ndarray):
    """mean_j |v_j| over the bodies and its bound, given per-body bounds e_j of the error of the kernel's fp32 vector."""
    val = _norm(v).mean(-1)
    return val, e.mean(-1) + 10 * U32 * val


def mpjpe_g(pred, gt):
    """Global MPJPE (also extras['mpjpe']): mean_j |p_j - g_j|."""
    p, g = _f64(pred), _f64(gt)
    d = p - g
    return _mean_norm(d, U32 * _norm(d))


def mpjpe_l(pred, gt):
    """Root-relative MPJPE: the root (body 0) subtracted from both poses."""
    p, g = _f64(pred), _f64(gt)
    y, x = p - p[:, :1], g - g[:, :1]
    l = y - x
    return _mean_norm(l, U32 * (_norm(y) + _norm(x) + _norm(l)))


def vel_dist(pred1, gt1, pred0, gt0):
    """compute_error_vel of frame t (pred1, gt1) after frame t - 1 (pred0, gt0): mean_j |(p1 - p0) - (g1 - g0)|.  The kernel differences
    the stored fp32 d = fl(p - g) of the two frames."""
    d1, d0 = _f64(pred1) - _f64(gt1), _f64(pred0) - _f64(gt0)
    v = d1 - d0
    return _mean_norm(v, U32 * (_norm(d1) + _norm(d0) + _norm(v)))


def accel_dist(pred2, gt2, pred1, gt1, pred0, gt0):
    """compute_error_accel ending at frame t (pred2, gt2): mean_j |(p2 - 2 p1 + p0) - (g2 - 2 g1 + g0)|."""
    d2, d1, d0 = _f64(pred2) - _f64(gt2), _f64(pred1) - _f64(gt1), _f64(pred0) - _f64(gt0)
    c = d2 - 2 * d1 + d0
    mag = _norm(d2) + 2 * _norm(d1) + _norm(d0)
    return _mean_norm(c, 3 * U32 * mag + U32 * _norm(c))


def p_mpjpe64(pred_rel: np.ndarray, gt_rel: np.ndarray) -> np.ndarray:
    """VideoPose3D p_mpjpe in float64 (centre, normalise, SVD, determinant sign fix, scale tr |X| / |Y|), [F, J, 3] x 2 -> [F]."""
    muX, muY = gt_rel.mean(1, keepdims=True), pred_rel.mean(1, keepdims=True)
    X0, Y0 = gt_rel - muX, pred_rel - muY
    nX = np.sqrt((X0 ** 2).sum((1, 2), keepdims=True))
    nY = np.sqrt((Y0 ** 2).sum((1, 2), keepdims=True))
    X0, Y0 = X0 / nX, Y0 / nY
    H = np.matmul(X0.transpose(0, 2, 1), Y0)
    U, s, Vt = np.linalg.svd(H)
    V = Vt.transpose(0, 2, 1)
    sd = np.sign(np.linalg.det(np.matmul(V, U.transpose(0, 2, 1))))
    V[:, :, -1] *= sd[:, None]
    s[:, -1] *= sd
    R = np.matmul(V, U.transpose(0, 2, 1))
    a = s.sum(1)[:, None, None] * nX / nY
    t = muX - a * np.matmul(muY, R)
    aligned = a * np.matmul(pred_rel, R) + t
    return _norm(aligned - gt_rel).mean(-1)


def horn_matrix(S: np.ndarray) -> np.ndarray:
    """Horn's 4x4 symmetric matrix of S[a][b] = sum_j Y_a X_b (its top eigenvector is the quaternion rotating Y onto X), [F, 3, 3]."""
    N = np.empty(S.shape[:-2] + (4, 4))
    N[..., 0, 0] = S[..., 0, 0] + S[..., 1, 1] + S[..., 2, 2]
    N[..., 1, 1] = S[..., 0, 0] - S[..., 1, 1] - S[..., 2, 2]
    N[..., 2, 2] = -S[..., 0, 0] + S[..., 1, 1] - S[..., 2, 2]
    N[..., 3, 3] = -S[..., 0, 0] - S[..., 1, 1] + S[..., 2, 2]
    N[..., 0, 1] = N[..., 1, 0] = S[..., 1, 2] - S[..., 2, 1]
    N[..., 0, 2] = N[..., 2, 0] = S[..., 2, 0] - S[..., 0, 2]
    N[..., 0, 3] = N[..., 3, 0] = S[..., 0, 1] - S[..., 1, 0]
    N[..., 1, 2] = N[..., 2, 1] = S[..., 0, 1] + S[..., 1, 0]
    N[..., 1, 3] = N[..., 3, 1] = S[..., 2, 0] + S[..., 0, 2]
    N[..., 2, 3] = N[..., 3, 2] = S[..., 1, 2] + S[..., 2, 1]
    return N


def quat_matrix(q: np.ndarray) -> np.ndarray:
    """R(q) for q = (w, x, y, z) (normalised here), [..., 4] -> [..., 3, 3]; R(q) Y rotates column vectors."""
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def horn64(X: np.ndarray, Y: np.ndarray) -> Dict[str, np.ndarray]:
    """Horn's method in float64 on centred sets [F, J, 3]: eigenvalues (descending) and eigenvectors of N, R, scale."""
    S = np.einsum("fja,fjb->fab", Y, X)
    N = horn_matrix(S)
    lam, vec = np.linalg.eigh(N)
    lam, vec = lam[:, ::-1], vec[:, :, ::-1]
    ny2 = (Y * Y).sum((1, 2))
    return {"S": S, "N": N, "lam": lam, "vec": vec, "R": quat_matrix(vec[:, :, 0]), "scale": lam[:, 0] / ny2, "ny2": ny2}


def pa_mpjpe(pred, gt) -> Dict[str, np.ndarray]:
    """Procrustes-aligned MPJPE of the root-relative poses: value (p_mpjpe definition), bound, Horn's relative eigen-gap, the
    near-tie mask; for near-tie frames `value` is the middle of the range over the tied eigenspace and `tol` its half-width + slack."""
    p, g = _f64(pred), _f64(gt)
    yr, xr = p - p[:, :1], g - g[:, :1]
    val = p_mpjpe64(yr, xr)
    X, Y = xr - xr.mean(1, keepdims=True), yr - yr.mean(1, keepdims=True)
    h = horn64(X, Y)
    lam = h["lam"]
    nX, nY = _norm(X), _norm(Y)                                   # [F, J]
    # rounding of the coordinates: root-relative difference, the mean (butterfly + fl(1/24)), the centring
    eX = U32 * (_norm(xr) + nX) + 8 * U32 * _norm(xr).mean(-1, keepdims=True)
    eY = U32 * (_norm(yr) + nY) + 8 * U32 * _norm(yr).mean(-1, keepdims=True)
    M = (nY * nX).sum(-1)
    dS = (eY * nX + nY * eX).sum(-1) + 6 * U32 * M
    nN = np.abs(lam).max(-1)
    E = 2 * dS + 8 * U32 * M + C_JACOBI * U32 * nN
    ny2 = h["ny2"]
    dny2 = (2 * (nY * eY).sum(-1) + 8 * U32 * ny2) / ny2
    lam1 = lam[:, 0]
    gap = lam1 - lam[:, 1]
    gap_rel = gap / np.maximum(np.abs(lam1), 1e-300)
    tie = (gap_rel < TIE_GAP) | (gap < 4 * E)
    s = h["scale"]
    ds = E / np.abs(lam1) + dny2 + U32
    sin_q = np.where(tie, 1.0, E / np.maximum(gap - E, 1e-300)) + C_JACOBI * U32
    dR = np.minimum(2.0, 2 * sin_q + 12 * U32)
    aligned = s[:, None, None] * np.einsum("fab,fjb->fja", h["R"], Y) - X
    na = _norm(aligned)
    e_a = s[:, None] * nY * (ds[:, None] + dR[:, None] + 7 * U32) + s[:, None] * eY + eX + U32 * na
    tol = e_a.mean(-1) + 10 * U32 * val
    half = np.zeros_like(val)
    if tie.any():
        idx = np.flatnonzero(tie)
        lo, hi = _tie_range(X[idx], Y[idx], h["vec"][idx], s[idx])
        # the rounding of everything but the rotation, the scale's spread over the tied pair, the grid slack
        e_round = (s[idx, None] * nY[idx] * (ds[idx, None] + 12 * U32 + 7 * U32) + s[idx, None] * eY[idx] + eX[idx]
                   + U32 * na[idx]).mean(-1) + 10 * U32 * hi
        spread = (gap[idx] + E[idx]) / ny2[idx] * nY[idx].mean(-1)
        sin_off = E[idx] / np.maximum(lam1[idx] - lam[idx, 2] - E[idx], 1e-300)
        slack = s[idx] * nY[idx].mean(-1) * (math.pi / TIE_GRID + 2 * sin_off + 2 * C_JACOBI * U32)
        val[idx] = 0.5 * (lo + hi)
        half[idx] = 0.5 * (hi - lo)
        tol[idx] = half[idx] + e_round + spread + slack
    return {"value": val, "tol": tol, "half": half, "gap_rel": gap_rel, "tie": tie, "R": h["R"], "scale": s}


def tie_excess(got: np.ndarray, pa: Dict[str, np.ndarray]) -> np.ndarray:
    """For the near-tie frames of `pa`: how far the kernel's value lies outside the range over the tied span, as a fraction of the
    slack around it (0 inside the range, 1 at the edge of the bound)."""
    t = pa["tie"]
    v, mid, tol = np.asarray(got, np.float64)[t], pa["value"][t], pa["tol"][t]
    lo, hi = mid - pa["half"][t], mid + pa["half"][t]
    return np.maximum(0.0, np.maximum(lo - v, v - hi)) / (tol - pa["half"][t])


def _tie_range(X, Y, vec, s):
    """min / max over phi in [0, pi) of mean_j |s R(cos phi v1 + sin phi v2) Y_j - X_j|, [T] each."""
    phi = np.arange(TIE_GRID) * (math.pi / TIE_GRID)
    lo, hi = np.empty(X.shape[0]), np.empty(X.shape[0])
    for b in range(0, X.shape[0], 64):
        sl = slice(b, b + 64)
        q = np.cos(phi)[None, :, None] * vec[sl, None, :, 0] + np.sin(phi)[None, :, None] * vec[sl, None, :, 1]
        R = quat_matrix(q)                                                     # [B, G, 3, 3]
        v = _norm(s[sl, None, None, None] * np.matmul(Y[sl, None], np.swapaxes(R, -1, -2)) - X[sl, None]).mean(-1)
        lo[sl], hi[sl] = v.min(-1), v.max(-1)
    return lo, hi


def frame_values(pred, gt, hist: Sequence = ()) -> Dict[str, Dict[str, np.ndarray]]:
    """All per-frame metrics of one step, [F, 24, 3] fp32 each.  hist = ((pred, gt) of step t - 1, (pred, gt) of step t - 2), as far
    as they exist; vel_dist / accel_dist are only returned when they do."""
    out = {}
    out["mpjpe_g"] = dict(zip(("value", "tol"), mpjpe_g(pred, gt)))
    out["mpjpe_l"] = dict(zip(("value", "tol"), mpjpe_l(pred, gt)))
    out["mpjpe_pa"] = pa_mpjpe(pred, gt)
    if len(hist) >= 1:
        out["vel_dist"] = dict(zip(("value", "tol"), vel_dist(pred, gt, *hist[0])))
    if len(hist) >= 2:
        out["accel_dist"] = dict(zip(("value", "tol"), accel_dist(pred, gt, *hist[0], *hist[1])))
    return out


def compute_metrics_lite_sums(pred_all: List[np.ndarray], gt_all: List[np.ndarray]) -> Dict[str, np.ndarray]:
    """compute_metrics_lite over per-sequence frame lists ([T_i, 24, 3] fp32 each, the frames the reference keeps, i.e. [:(n - 1)]) as
    the kernel accumulates it: sums [N, 5] (metres, METRICS order), counts [N, 3] (frames, velocity frames, acceleration frames) and
    the bound of each sum (the per-frame bounds added up)."""
    n = len(pred_all)
    sums, tols = np.zeros((n, 5)), np.zeros((n, 5))
    counts = np.zeros((n, 3), dtype=np.int64)
    for i, (p, g) in enumerate(zip(pred_all, gt_all)):
        T = p.shape[0]
        counts[i] = (T, max(T - 1, 0), max(T - 2, 0))
        if T == 0:
            continue
        for k, (v, t) in enumerate((mpjpe_g(p, g), mpjpe_l(p, g))):
            sums[i, k], tols[i, k] = v.sum(), t.sum()
        pa = pa_mpjpe(p, g)
        sums[i, 2], tols[i, 2] = pa["value"].sum(), pa["tol"].sum()
        if T >= 2:
            v, t = vel_dist(p[1:], g[1:], p[:-1], g[:-1])
            sums[i, 3], tols[i, 3] = v.sum(), t.sum()
        if T >= 3:
            v, t = accel_dist(p[2:], g[2:], p[1:-1], g[1:-1], p[:-2], g[:-2])
            sums[i, 4], tols[i, 4] = v.sum(), t.sum()
    return {"sums": sums, "counts": counts, "tol": tols}


# ------------------------------------------------------------------------------------------------------------------------ frame classes
FRAME_CLASSES = ("rot_uniform", "rot_near_pi", "similarity", "mirror", "mirror_rot", "mirror_tie", "collinear", "coplanar", "scale",
                 "identical", "tiny", "far", "walk")


def _random_rotation(rng, angle=None) -> np.ndarray:
    """A rotation uniform over SO(3), or about a uniform axis by `angle`."""
    if angle is None:
        q = rng.normal(size=4)
        return quat_matrix(q / np.linalg.norm(q))
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    h = 0.5 * angle
    return quat_matrix(np.concatenate([[math.cos(h)], math.sin(h) * ax]))


def make_sequence(cls: str, rng, T: int):
    """T frames of one frame class: (pred, gt) fp32 [T, 24, 3].  The target is a pose with a drifting root and a slow per-body random
    walk; the prediction is the class's transform of it (fixed over the sequence) plus per-frame noise."""
    root = rng.normal(size=3) + np.cumsum(rng.normal(scale=0.03, size=(T, 3)), 0)
    if cls == "collinear":
        d = rng.normal(size=3)
        off = (rng.normal(scale=0.4, size=24)[None, :] + np.cumsum(rng.normal(scale=0.01, size=(T, 24)), 0))[..., None] * d / np.linalg.norm(d)
    else:
        off = rng.normal(scale=0.3, size=(1, 24, 3)) + np.cumsum(rng.normal(scale=0.01, size=(T, 24, 3)), 0)
        if cls == "mirror_tie":                         # principal moments (a, b, b): a mirror image ties Horn's top eigenvalues
            u, _, vt = np.linalg.svd(off[0] - off[0].mean(0), full_matrices=False)
            c = (u * np.array([0.5, 0.25, 0.25]) * math.sqrt(24)) @ vt
            off = np.broadcast_to(c - c[0], off.shape).copy()
        if cls == "coplanar":
            off = off @ np.linalg.qr(rng.normal(size=(3, 3)))[0][:, :2] @ np.linalg.qr(rng.normal(size=(3, 3)))[0][:2, :]
    off[:, 0] = 0.0
    if cls == "far":
        d = rng.normal(size=3)
        root = root + 10 ** rng.uniform(2, 3) * d / np.linalg.norm(d)
    gt = root[:, None, :] + off
    noise = 0.01 * rng.normal(size=(T, 24, 3))
    R, s, t = _random_rotation(rng), 1.0, rng.normal(size=3)
    if cls == "rot_uniform":
        R = _random_rotation(rng, rng.uniform(0, math.pi))
    elif cls == "rot_near_pi":
        R = _random_rotation(rng, math.pi - 10 ** rng.uniform(-7, -3))
    elif cls == "similarity":
        s, noise = 10 ** rng.uniform(-1, 1), 0 * noise
    elif cls == "mirror":
        R, t = np.diag([1.0, 1.0, -1.0]), np.zeros(3)
        noise = noise * 0.3 * rng.integers(0, 2)
    elif cls == "mirror_tie":
        R = R @ np.diag([1.0, 1.0, -1.0])
        noise = 1e-4 * noise * rng.integers(0, 2)
    elif cls == "mirror_rot":
        R = R @ np.diag([1.0, 1.0, -1.0])
    elif cls == "scale":
        s = 10 ** rng.uniform(-1, 1)
        noise = noise * s
    elif cls in ("identical", "tiny", "far", "walk"):
        R, t = np.eye(3), np.zeros(3)
        if cls == "identical":
            noise = 0 * noise
        elif cls == "tiny":
            noise = 1e-3 * noise
        elif cls == "walk":
            noise = np.cumsum(0.004 * rng.normal(size=(T, 24, 3)), 0) + noise
    if cls == "far":
        R = _random_rotation(rng, rng.uniform(0, 0.3))
        pred = root[:, None, :] + s * off @ R.T + noise
    else:
        pred = s * gt @ R.T + t + noise
    gt32 = gt.astype(np.float32)
    pred32 = gt32.copy() if cls == "identical" else pred.astype(np.float32)
    return pred32, gt32


def means_mm(sums: np.ndarray, counts: np.ndarray, tol: np.ndarray, select: Optional[np.ndarray] = None):
    """np.mean over the concatenated per-frame arrays, in mm, and its bound: (values, bounds) dicts keyed by METRICS."""
    if select is not None:
        sums, counts, tol = sums[select], counts[select], tol[select]
    col = (0, 0, 0, 1, 2)
    val, bnd = {}, {}
    for k, name in enumerate(METRICS):
        c = counts[:, col[k]].sum()
        val[name] = sums[:, k].sum() / c * 1000.0 if c > 0 else float("nan")
        bnd[name] = tol[:, k].sum() / c * 1000.0 if c > 0 else float("nan")
    return val, bnd
