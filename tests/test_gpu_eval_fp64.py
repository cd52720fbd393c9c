"""pulse_eval_step frame by frame against the float64 reference of tests/eval_fp64.py.

One env per case, the frame classes of `eval_fp64.FRAME_CLASSES` (random rotations over [0, pi] and near pi, exact similarity
transforms, mirror images with and without rotation, mirrored poses with tied principal moments, collinear and coplanar body sets,
scales 0.1 .. 10, pred == gt bit for bit, 1e-5 m errors, roots 10^2 .. 10^3 m away, the synthetic walk of test_gpu_eval.py) spread
over the envs.  After every step the test synchronises and reads the state: each env's increment of the fp64 sums is that frame's
value (to within u64 of the running sum), held to the reference's bound; counts, terminate_state, ctrl and extras['mpjpe'] follow
`EvalOracle.post_step` step by step; once the chunk has ended further steps change no buffer.  Run with -s for the margin report."""
import numpy as np
import pytest
import torch

from oracle.eval_oracle import EvalOracle
from tests import eval_fp64 as ef
from tests.fp64_ref import Report

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EXACT_ZERO = {"identical": ("mpjpe_g", "mpjpe_l", "vel_dist", "accel_dist")}


class _Margins:
    """Largest |kernel - fp64| / bound per (frame class, metric), near-tie frames counted apart."""

    def __init__(self):
        self.worst, self.ties, self.tie_excess, self.frames = {}, {}, {}, {}

    def add(self, cls_of, metric, got, ref, tol, tie=None, excess=None):
        err = np.abs(got - ref)
        r = np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), np.where(err > 0, np.inf, 0.0))
        plain = np.ones_like(r, dtype=bool) if tie is None else ~tie
        for c in np.unique(cls_of):
            m = cls_of == c
            key = (c, metric)
            if (m & plain).any():                          # near-tie frames are reported by how far they leave the tied range
                self.worst[key] = max(self.worst.get(key, 0.0), float(r[m & plain].max()))
            self.frames[key] = self.frames.get(key, 0) + int(m.sum())
            if tie is not None:
                self.ties[c] = self.ties.get(c, 0) + int(tie[m].sum())
                if excess is not None and (tie & m).any():
                    self.tie_excess[c] = max(self.tie_excess.get(c, 0.0), float(excess[m[tie]].max()))
        bad = np.flatnonzero(~(r < 1.0))
        if bad.size:
            k = bad[0]
            raise AssertionError(f"{metric} [{cls_of[k]}]: {bad.size} frames over the bound, first env {k}: kernel {got[k]!r}, "
                                 f"fp64 {ref[k]!r}, bound {tol[k]:.3e}, err/tol {r[k]:.3f}")

    def report(self, title):
        rep = Report(title)
        for (c, metric) in sorted(self.frames):
            r, exc = self.worst.get((c, metric), 0.0), None
            if metric == "mpjpe_pa" and self.ties.get(c):
                exc = (f"{self.ties[c]} of {self.frames[(c, metric)]} frames near-tied (gap < {ef.TIE_GAP:g}), checked against the "
                       f"range over the tied span: worst excess {self.tie_excess.get(c, 0.0):.4f}")
            rep.add(f"{c} / {metric}", r, excluded=exc)
        return rep.text()


def _scene(N, S, seed, offset=0):
    rng = np.random.default_rng(seed)
    cls = np.array([ef.FRAME_CLASSES[(e + offset) % len(ef.FRAME_CLASSES)] for e in range(N)])
    pred, gt = np.empty((S, N, 24, 3), np.float32), np.empty((S, N, 24, 3), np.float32)
    for e in range(N):
        pred[:, e], gt[:, e] = ef.make_sequence(cls[e], rng, S)
    return cls, pred, gt


class _Views:
    """The simulator's [N, 26, 13] rigid-body state and the reference positions, contiguous or as a [N, 24, 4][..., :3] view."""

    def __init__(self, N, strided_gt):
        self.state = torch.zeros(N, 26, 13, device=DEV)
        self.gt_store = torch.zeros(N, 24, 4 if strided_gt else 3, device=DEV)
        self.term = torch.zeros(N, dtype=torch.int64, device=DEV)

    def load(self, pred, gt, term):
        self.state[:, :24, :3].copy_(torch.from_numpy(pred))
        self.gt_store[..., :3].copy_(torch.from_numpy(gt))
        self.term.copy_(torch.from_numpy(term.astype(np.int64)))
        return self.state, self.gt_store[..., :3], self.term


def _snapshot(m):
    torch.cuda.synchronize()
    return {k: getattr(m, k).clone() for k in ("sums", "counts", "terminate_state", "ctrl", "mpjpe", "hist")}


def _run_chunk(m, orc, views, margins, cls, pred, gt, num_steps, ids, fail_step, garbage_hist=False):
    """Drives one chunk step by step, checking every step; returns the steps taken, the final terminate_state and the final buffers."""
    N = len(num_steps)
    bound = N if (ids != orc.num_unique - 1).all() else int(np.flatnonzero(ids == orc.num_unique - 1)[0]) + 1
    m.begin_chunk(num_steps, bound)
    if garbage_hist:                                       # no value of the chunk may depend on the history it starts with
        m.hist.copy_(torch.tensor([np.nan, 3e38, -1e30], device=DEV).repeat(m.hist.numel() // 3).view_as(m.hist))
    prev = _snapshot(m)
    counts = np.zeros((N, 3), np.int64)
    k, finished = 0, False
    while not finished:
        term = fail_step == k
        m.step(*views.load(pred[k], gt[k], term))
        cur = _snapshot(m)
        s = {n: t.cpu().numpy() for n, t in cur.items()}
        ds = s["sums"] - prev["sums"].cpu().numpy()
        slack = 2 * ef.U64 * np.abs(s["sums"])
        mg = ef.mpjpe_g(pred[k], gt[k])
        margins.add(cls, "extras_mpjpe", s["mpjpe"].astype(np.float64), mg[0], mg[1])
        chunk_done, end, info = orc.post_step(term, s["mpjpe"], pred[k], gt[k], num_steps, ids)
        finished = chunk_done or end
        term_ref = orc.terminate_memory[-1] if finished else orc.terminate_state
        np.testing.assert_array_equal(s["terminate_state"].astype(bool), term_ref, err_msg=f"terminate_state after step {k}")
        assert s["ctrl"][0] == k + 1 and s["ctrl"][1] == int(finished) and not s["ctrl"][2:5].any(), (k, s["ctrl"])
        counted = k < num_steps - 1
        counts += counted[:, None] * np.array([1, k >= 1, k >= 2])
        np.testing.assert_array_equal(s["counts"], counts, err_msg=f"counts after step {k}")
        hist = [(pred[k - i], gt[k - i]) for i in (1, 2) if k - i >= 0]
        ref = ef.frame_values(pred[k], gt[k], hist)
        for c, name in enumerate(ef.METRICS):
            col_counted = counted & (k >= (0, 0, 0, 1, 2)[c])
            assert (ds[~col_counted, c] == 0).all(), (name, k)          # frames outside [:(n - 1)] add nothing
            if name not in ref or not col_counted.any():
                continue
            r = ref[name]
            sel = col_counted
            tie = r.get("tie")
            sub = {q: r[q][sel] for q in ("value", "tol", "half", "tie") if q in r}
            margins.add(cls[sel], name, ds[sel, c], sub["value"], sub["tol"] + slack[sel, c], tie=sub.get("tie"),
                        excess=ef.tie_excess(ds[sel, c], sub) if "tie" in sub else None)
            for zc, names in EXACT_ZERO.items():
                z = sel & (cls == zc)
                if name in names and z.any():
                    assert (ds[z, c] == 0).all(), (name, zc, k)
        if "mpjpe_pa" in ref and counted.any():
            assert np.isfinite(ds[:, 2]).all()
        prev = cur
        k += 1
    frozen = _snapshot(m)
    for extra in range(2):                                 # the chunk has ended: further launches change nothing
        m.step(*views.load(pred[k + extra], gt[k + extra], np.ones(N, bool)))
        after = _snapshot(m)
        for n in frozen:
            assert torch.equal(after[n].nan_to_num(), frozen[n].nan_to_num()) and torch.equal(after[n].isnan(), frozen[n].isnan()), n
    return k, frozen["terminate_state"].cpu().numpy().astype(bool), frozen


@pytest.mark.parametrize("N,strided_gt", [(1, False), (3, True), (1027, True), (1027, False), (16384, True)])
def test_frames_by_class(N, strided_gt):
    from pulse_b200.evaluation import EvalMetricsB200
    rng = np.random.default_rng(N)
    num_steps = rng.choice([1, 2, 3, 4, 5, 9, 14] if N < 16384 else [1, 2, 3, 4, 6], size=N)
    if N <= 3:
        num_steps[:] = [4, 1, 2][:N] if N == 3 else 6
    S = int(num_steps.max()) + 4
    cls, pred, gt = _scene(N, S, seed=100 + N, offset=N)
    fail_step = np.where(rng.random(N) < 0.3, rng.integers(0, S, size=N), 10 ** 6)
    m, views, margins = EvalMetricsB200(N, DEV), _Views(N, strided_gt), _Margins()
    orc = EvalOracle(N, 10 * N, np.array([f"c{i}" for i in range(10 * N)]))
    _run_chunk(m, orc, views, margins, cls, pred, gt, num_steps, np.arange(N), fail_step)
    print("\n" + margins.report(f"pulse_eval_step vs fp64, N={N}, body_pos_gt {'strided' if strided_gt else 'contiguous'}"))


@pytest.mark.parametrize("N,U", [(1027, 2033), (64, 100)])
def test_wrapped_second_chunk_and_readout(N, U):
    """Two chunks with the EvalOracle carried across: the second wraps (bound < N) and starts from a history full of garbage.  The
    host's `summarise` over the read-back sums equals the fp64 compute_metrics_lite means over the first U sequences (all and the
    successful subset), in mm, within the propagated bound."""
    from pulse_b200.evaluation import EvalMetricsB200, summarise
    rng = np.random.default_rng(U)
    m, views, margins = EvalMetricsB200(N, DEV), _Views(N, True), _Margins()
    keys = np.array([f"c{i}" for i in range(U)])
    orc = EvalOracle(N, U, keys)
    steps_all = rng.choice([1, 2, 3, 4, 6, 11], size=U)
    fail_all = np.where(rng.random(U) < 0.4, rng.integers(0, 12, size=U), 10 ** 6)
    sums, counts, terms, P, G = [], [], [], [], []
    for chunk in range(2):
        ids = (chunk * N + np.arange(N)) % U
        num_steps = steps_all[ids]
        S = int(num_steps.max()) + 4
        cls, pred, gt = _scene(N, S, seed=7 * U + chunk, offset=chunk)
        taken, term, fin = _run_chunk(m, orc, views, margins, cls, pred, gt, num_steps, ids, fail_all[ids], garbage_hist=chunk == 1)
        sums.append(fin["sums"].cpu().numpy()); counts.append(fin["counts"].cpu().numpy()); terms.append(term)
        P += [pred[:min(taken, n - 1), e] for e, n in enumerate(num_steps)]
        G += [gt[:min(taken, n - 1), e] for e, n in enumerate(num_steps)]
    assert orc.start_idx + N >= U
    sums, counts, term = np.concatenate(sums)[:U], np.concatenate(counts)[:U], np.concatenate(terms)[:U]
    ref = ef.compute_metrics_lite_sums(P[:U], G[:U])
    np.testing.assert_array_equal(counts, ref["counts"])
    for select in (None, ~term):
        got = summarise(sums, counts, select)
        want, bnd = ef.means_mm(ref["sums"], ref["counts"], ref["tol"], select)
        for k in ef.METRICS:
            assert np.isnan(got[k]) == np.isnan(want[k]), k
            assert np.isnan(want[k]) or abs(got[k] - want[k]) <= bnd[k] + 1e-12 * abs(want[k]), (k, select is None, got[k], want[k], bnd[k])
    print("\n" + margins.report(f"two chunks, N={N}, U={U} (wrapped second chunk)"))


class _ClassSim:
    """A MotionLib / task stand-in for EvalLoopB200 whose clips are frame-class sequences."""

    def __init__(self, N, U, seed, fail_all=False):
        self.N, self.U, self.seed = N, U, seed
        rng = np.random.default_rng(seed)
        self.steps = rng.choice([2, 3, 5, 8], size=U)
        self.fail = rng.integers(0, 2, size=U) if fail_all else np.where(rng.random(U) < 0.5, rng.integers(0, 9, size=U), 10 ** 6)
        self.keys = np.array([f"clip{i}" for i in range(U)])
        self.frames, self.taken = [], []

    def load_chunk(self, start):
        self.ids = (start + np.arange(self.N)) % self.U
        self.s = 0
        self.taken.append(0)
        self.cls, self.pred, self.gt = _scene(self.N, int(self.steps[self.ids].max()) + 12, self.seed + start, start)
        self.frames.append((self.pred, self.gt, self.steps[self.ids]))
        return self.steps[self.ids], self.ids


@pytest.mark.parametrize("fail_all", [False, True])
def test_eval_loop_readout_against_fp64(fail_all):
    """EvalLoopB200 end to end: success-subset selection, and the fallback to all sequences when none succeeded."""
    from pulse_b200.evaluation import EvalLoopB200
    N, U = 48, 80
    sim = _ClassSim(N, U, 5, fail_all)
    v = _Views(N, False)

    def step():
        k = min(sim.s, sim.pred.shape[0] - 1)
        sim.s += 1
        sim.taken[-1] = sim.s
        return v.load(sim.pred[k], sim.gt[k], sim.fail[sim.ids] == k)

    out = EvalLoopB200(N, U, sim.keys, load_chunk=sim.load_chunk, reset_all=lambda: None, step=step, device=DEV, poll_every=1).run()
    term = out["terminated"]
    assert term.all() == fail_all
    P, G = [], []
    for (pred, gt, ns), taken in zip(sim.frames, sim.taken):            # a chunk in which every env failed ends early
        P += [pred[:min(taken, n - 1), e] for e, n in enumerate(ns)]
        G += [gt[:min(taken, n - 1), e] for e, n in enumerate(ns)]
    ref = ef.compute_metrics_lite_sums(P[:U], G[:U])
    np.testing.assert_array_equal(out["per_sequence"]["counts"], ref["counts"])
    all_v, all_b = ef.means_mm(ref["sums"], ref["counts"], ref["tol"])
    succ_v, succ_b = ef.means_mm(ref["sums"], ref["counts"], ref["tol"], ~term) if (~term).any() else (all_v, all_b)
    info = out["eval_info"]
    pairs = {"eval_mpjpe_all": (all_v, all_b, "mpjpe_g"), "mpjpel_all": (all_v, all_b, "mpjpe_l"),
             "eval_mpjpe_succ": (succ_v, succ_b, "mpjpe_g"), "mpjpel_succ": (succ_v, succ_b, "mpjpe_l"),
             "mpjpe_pa": (succ_v, succ_b, "mpjpe_pa"), "vel_dist": (succ_v, succ_b, "vel_dist"), "accel_dist": (succ_v, succ_b, "accel_dist")}
    for name, (vals, bnds, k) in pairs.items():
        if np.isnan(vals[k]):                                  # no frame of that kind in the selection (a chunk that ended early)
            assert np.isnan(info[name]), name
            continue
        assert abs(info[name] - vals[k]) <= bnds[k] + 1e-12 * abs(vals[k]), (name, info[name], vals[k], bnds[k])
    assert abs(info["eval_success_rate"] - (1 - term.mean())) < 1e-12
