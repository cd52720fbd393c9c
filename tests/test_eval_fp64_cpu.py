"""The float64 evaluation reference (tests/eval_fp64.py) checked on its own, without a GPU: properties of the Procrustes definition,
a brute-force optimum for mirror images, two independent constructions of the optimal rotation (one of them Horn's, which pins the
kernel's convention), and agreement with the fp32 restatement in oracle/eval_oracle.py within its rounding."""
import math

import numpy as np
import pytest
from scipy.linalg import orthogonal_procrustes
from scipy.optimize import minimize
from scipy.spatial.transform import Rotation

from oracle import eval_oracle as eo
from tests import eval_fp64 as ef


def _pose(rng, F=1):
    x = rng.normal(scale=0.3, size=(F, 24, 3))
    return x - x[:, :1]


def _rotations(rng, F, near_pi=False):
    if not near_pi:
        return Rotation.random(F, random_state=int(rng.integers(1 << 30))).as_matrix()
    ax = rng.normal(size=(F, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    return Rotation.from_rotvec(ax * (math.pi - 10 ** rng.uniform(-9, -3, size=(F, 1)))).as_matrix()


@pytest.mark.parametrize("near_pi", [False, True])
def test_similarity_transforms_vanish(near_pi):
    rng = np.random.default_rng(1 + near_pi)
    F = 256
    gt = _pose(rng, F)
    R = _rotations(rng, F, near_pi)
    s = 10 ** rng.uniform(-1, 1, size=(F, 1, 1))
    pred = s * np.einsum("fab,fjb->fja", R, gt) + rng.normal(scale=5.0, size=(F, 1, 3))
    pa = ef.p_mpjpe64(pred - pred[:, :1], gt)
    assert pa.max() < 1e-12 * np.abs(gt).max()
    X, Y = gt - gt.mean(1, keepdims=True), pred - pred.mean(1, keepdims=True)
    h = ef.horn64(X, Y)
    np.testing.assert_allclose(h["R"], np.transpose(R, (0, 2, 1)), atol=1e-9)   # Y was s R X: Horn rotates it back
    np.testing.assert_allclose(h["scale"], 1.0 / s[:, 0, 0], rtol=1e-12)


def _brute_force_pa(Y, X, starts):
    """min over proper rotations (rotation vector) of the least-squares objective with the optimal scale >= 0, several starts; the mean
    distance at the best optimum."""
    def aligned(r):
        RY = Y @ Rotation.from_rotvec(r).as_matrix().T
        return max((RY * X).sum(), 0.0) / (Y * Y).sum() * RY          # a negative scale would be a point reflection

    best = min((minimize(lambda r: ((aligned(r) - X) ** 2).sum(), r0, method="BFGS", options={"gtol": 1e-12}) for r0 in starts),
               key=lambda o: o.fun)
    return np.linalg.norm(aligned(best.x) - X, axis=-1).mean(), Rotation.from_rotvec(best.x).as_matrix()


@pytest.mark.parametrize("rotate", [False, True])
def test_mirror_image_matches_brute_force(rotate):
    rng = np.random.default_rng(7 + rotate)
    for _ in range(6):
        gt = _pose(rng)[0]
        pred = gt * np.array([1.0, 1.0, -1.0])
        if rotate:
            pred = pred @ _rotations(rng, 1)[0].T
        pred = pred + rng.normal(scale=0.005, size=pred.shape)
        X, Y = gt - gt.mean(0), pred - pred.mean(0)
        starts = [np.zeros(3)] + [Rotation.random(random_state=int(rng.integers(1 << 30))).as_rotvec() for _ in range(7)]
        want, R = _brute_force_pa(Y, X, starts)
        got = ef.p_mpjpe64((pred - pred[:1])[None], (gt - gt[:1])[None])[0]
        assert abs(got - want) <= 1e-7 * want, (got, want)
        np.testing.assert_allclose(ef.horn64(X[None], Y[None])["R"][0], R, atol=1e-5)
        # the unconstrained optimum is the reflection, which p_mpjpe must not use
        assert np.linalg.det(orthogonal_procrustes(Y, X)[0]) < 0


def test_rotation_agrees_with_orthogonal_procrustes_and_horn():
    rng = np.random.default_rng(3)
    for cls in ("rot_uniform", "rot_near_pi", "mirror_rot", "coplanar", "scale", "walk"):
        for _ in range(8):
            p, g = ef.make_sequence(cls, rng, 1)
            p, g = p[0].astype(np.float64), g[0].astype(np.float64)
            X, Y = g - g.mean(0), p - p.mean(0)
            # orthogonal_procrustes: argmin |Y Q - X| over orthogonal Q (row vectors); the sign fix makes Q proper
            u, _, vt = np.linalg.svd(Y.T @ X)
            d = np.sign(np.linalg.det(u @ vt))
            Q = u @ np.diag([1.0, 1.0, d]) @ vt
            if d > 0:
                np.testing.assert_allclose(Q, orthogonal_procrustes(Y, X)[0], atol=1e-10)
            h = ef.horn64(X[None], Y[None])
            np.testing.assert_allclose(h["R"][0], Q.T, atol=1e-8)             # Horn: S[a][b] = sum_j Y_a X_b, R(q) Y rotated onto X
            S_t = np.einsum("ja,jb->ab", X, Y)                                  # the transposed correlation gives R^T, not R
            R_t = ef.quat_matrix(np.linalg.eigh(ef.horn_matrix(S_t))[1][:, -1])
            if cls in ("rot_uniform", "mirror_rot", "scale"):            # (a rotation by 0 or pi is its own transpose)
                assert np.abs(R_t - Q.T).max() > 1e-3
            # the value from either rotation is p_mpjpe's
            s = h["scale"][0]
            v_h = np.linalg.norm(s * Y @ h["R"][0].T - X, axis=-1).mean()
            v_p = ef.p_mpjpe64((p - p[:1])[None], (g - g[:1])[None])[0]
            assert abs(v_h - v_p) <= 1e-10 * max(v_p, 1e-3)


def test_near_ties_are_flagged():
    rng = np.random.default_rng(5)
    seq = {c: [ef.make_sequence(c, rng, 1) for _ in range(16)] for c in ("collinear", "mirror_tie", "rot_uniform", "coplanar")}
    flag = {c: ef.pa_mpjpe(np.concatenate([p for p, _ in v]), np.concatenate([g for _, g in v]))["tie"] for c, v in seq.items()}
    assert flag["collinear"].all() and flag["mirror_tie"].all()
    assert not flag["rot_uniform"].any() and not flag["coplanar"].any()


def test_reference_refuses_fp64_input():
    with pytest.raises(TypeError):
        ef.mpjpe_g(np.zeros((1, 24, 3)), np.zeros((1, 24, 3)))


def test_fp32_restatement_agrees_within_rounding():
    """oracle.eval_oracle evaluates the same definitions on fp32 arrays (numpy's fp32 SVD, norms, means): it agrees with the float64
    reference within the same bounds, class by class."""
    rng = np.random.default_rng(11)
    for cls in ef.FRAME_CLASSES:
        P, G = zip(*[ef.make_sequence(cls, rng, 1) for _ in range(32)])
        P, G = np.concatenate(P), np.concatenate(G)
        pa = ef.pa_mpjpe(P, G)
        got = eo.p_mpjpe(P - P[:, :1], G - G[:, :1]).astype(np.float64)
        assert got.dtype == np.float64
        ok = ~pa["tie"]
        err = np.abs(got - pa["value"])[ok]
        assert (err <= pa["tol"][ok]).all(), (cls, float((err / pa["tol"][ok]).max()))
        assert (np.abs(got - pa["value"]) <= pa["tol"] + 2 * pa["half"]).all(), cls


def test_sequence_oracle_matches_compute_metrics_lite():
    rng = np.random.default_rng(13)
    lens = [0, 1, 2, 3, 4, 9]
    classes = ("rot_uniform", "rot_near_pi", "similarity", "mirror", "mirror_rot", "walk")     # no near ties: values are p_mpjpe's
    seqs = [ef.make_sequence(classes[i], rng, T) if T else
            (np.zeros((0, 24, 3), np.float32), np.zeros((0, 24, 3), np.float32)) for i, T in enumerate(lens)]
    P, G = [p for p, _ in seqs], [g for _, g in seqs]
    r = ef.compute_metrics_lite_sums(P, G)
    np.testing.assert_array_equal(r["counts"], [[0, 0, 0], [1, 0, 0], [2, 1, 0], [3, 2, 1], [4, 3, 2], [9, 8, 7]])
    val, bnd = ef.means_mm(r["sums"], r["counts"], r["tol"])
    keep = [i for i, T in enumerate(lens) if T > 0]
    m = eo.compute_metrics_lite([P[i].astype(np.float64) for i in keep], [G[i].astype(np.float64) for i in keep])
    for k in ef.METRICS:
        assert abs(np.mean(m[k]) - val[k]) <= 1e-9 * abs(val[k]), k
        assert 0 < bnd[k] < 1e-3 * abs(val[k]), k
    sel = np.array([True, False, True, True, False, True])
    v2, _ = ef.means_mm(r["sums"], r["counts"], r["tol"], sel)
    m2 = eo.compute_metrics_lite([P[i].astype(np.float64) for i in (2, 3, 5)], [G[i].astype(np.float64) for i in (2, 3, 5)])
    for k in ef.METRICS:
        assert abs(np.mean(m2[k]) - v2[k]) <= 1e-9 * abs(v2[k]), k
