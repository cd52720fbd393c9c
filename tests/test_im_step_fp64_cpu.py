"""The imitation step's float64 references (tests/step_fp64.py: im_step_ref, task_obs_ref) have teeth: a float32 CPU simulation of
im_step_kernel and of task_obs_kernel passes every link, and a simulation with one defect fails the link it breaks with BoundError
naming it.  The simulations restate the kernels' arithmetic (im_step.cu, task_obs.cu, quat_math.cuh) in float32 torch operations, with
the pinned fp32 order wherever the kernel's result decides an integer (motion times, frame rows, the termination distance).
The input generators (with the built edge envs) are shared with tests/test_gpu_im_step_fp64.py."""
import dataclasses
import math
import re
from types import SimpleNamespace

import pytest
import torch

from oracle import pulse_oracle as po
from tests import step_fp64 as sf
from tests.helpers import exact_tables, synthetic_step_inputs
from tests.test_motion_fp64_cpu import expmap32, qmul8_32, slerp32
from tests.test_reset_fp64_cpu import qrot32, six32
from tests.test_task_step_fp64_cpu import base_removed32, heading_half32, self_obs32

MIXED_RATES = (24.0, 25.0, 29.97, 30.0, 50.0, 60.0, 120.0)
DEFAULT_RESET_BODIES = tuple(j for j in range(24) if j not in (3, 4, 7, 8))
BUILT = 24                      # rows 0 .. BUILT - 1 of a generated batch are the built edge envs
ON_POSE, VERTICAL, FLIPPED, NEAR_PI, AT_PI = 0, 1, 2, 3, 4
PROG1, PROG2, PROG3, PROG4 = 5, 6, 7, 8
AT_LEN, BELOW_LEN, ON_FRAME, PAST_END, ONE_FRAME, TWO_FRAMES = 9, 10, 11, 12, 13, 14
CYC_PASS, CYC_HOLD, RECOVERING = 15, 16, 17
AT_TERM, PAST_TERM, UNMASKED_FAR = 18, 19, 20


def mask_of(ids) -> int:
    m = 0
    for j in ids:
        m |= 1 << int(j)
    return m


# ---------------------------------------------------------------------------------------------------------------- inputs
def im_tables(M: int, seed: int, fps=30.0):
    """exact_tables with clip 0 of 2 frames and clip 1 of 1 frame (its length 0); the rows past clip 1's frame stay in the tables."""
    tb = exact_tables(M, seed=seed, fps=fps)
    tb.num_frames = tb.num_frames.clone()
    tb.num_frames[1] = 1
    tb.lengths = tb.lengths.clone()
    tb.lengths[1] = 0.0
    return tb


def table_dict(tb):
    return {k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames", "dt",
                                        "length_starts", "fps", "motion_bodies", "motion_limb_weights")}


def config(**kw):
    """The ImConfig fields the step reads, with the step's termination distances and reset mask."""
    from pulse_b200.humanoid_im import ImConfig
    term = kw.pop("term", None)
    mask = kw.pop("mask", mask_of(DEFAULT_RESET_BODIES))
    c = ImConfig(**kw)
    c.term = torch.full((24,), float(c.termination_distance)) if term is None else term.float()
    c.mask = mask
    return c


def nonuniform_term():
    """Per-body termination distances: 0.25 for the bodies the built threshold rows use, others 0.15 .. 0.35, body 0 0.6."""
    t = 0.15 + 0.05 * (torch.arange(24) % 5).float()
    t[0] = 0.6
    return t


def _time_at(target: float, pd: torch.Tensor) -> float:
    """A start time s with fp32(pd + s) == target (pd fp32)."""
    tg = torch.tensor(target, dtype=torch.float32)
    s = (tg - pd).reshape(1)
    for _ in range(64):
        t = (pd + s)[0]
        if t == tg:
            return float(s[0])
        s = torch.nextafter(s, torch.full_like(s, math.inf if t < tg else -math.inf))
    raise AssertionError("no start time reaches the target")


def im_inputs(tb, n: int, seed: int, cfg, flags: int = 7, power: bool = True, recovery: bool = False):
    """Inputs of one step (CPU), rows 0 .. BUILT - 1 the built edge envs when n >= BUILT."""
    z = synthetic_step_inputs(dataclasses.replace(tb, lengths=tb.lengths.clamp_min(1e-3)), n, seed=seed)   # the 1-frame clip: no 0 / 0
    inp = dict(body=z["body_state"].clone(), progress=z["progress_buf"].clone(), motion_ids=z["motion_ids"].clone(),
               start=z["start_times"].clone(), offset=z["start_offset"].clone(), goff=z["global_offset"].clone(),
               cycle=z["cycle_counter"].clone(), dof_force=z["dof_force"] if power else None, dof_vel=z["dof_vel"], flags=flags,
               term=cfg.term, mask=cfg.mask, recovery=None)
    g = torch.Generator().manual_seed(seed + 7)
    if recovery:
        inp["recovery"] = (torch.rand(n, generator=g) < 0.3).int() * torch.randint(1, 100, (n,), generator=g, dtype=torch.int32)
    if n >= BUILT:
        _build_edges(tb, inp, cfg)
    return inp


def _pose(tb, ids, t, goff):
    ms = po.motion_state(tb, ids, t, goff)
    return torch.cat([ms["rg_pos"], torch.nn.functional.normalize(ms["rb_rot"], dim=-1), ms["body_vel"], ms["body_ang_vel"]], -1)


def _build_edges(tb, inp, cfg):
    body, prog, ids, start, off, goff, cyc = (inp[k] for k in ("body", "progress", "motion_ids", "start", "offset", "goff", "cycle"))
    dt32 = torch.tensor(cfg.dt, dtype=torch.float32)
    long_clip = int(torch.argmax(tb.num_frames[2:])) + 2
    B = slice(0, BUILT)
    ids[B], prog[B], off[B], cyc[B], goff[B] = long_clip, 10, 0.0, 0, 0.0
    ids[ONE_FRAME], ids[TWO_FRAMES] = 1, 0
    if inp["recovery"] is not None:
        inp["recovery"][B] = 0
        inp["recovery"][RECOVERING] = 20
    L, mdt = tb.lengths[long_clip], tb.dt[long_clip]
    adv = 1 if inp["flags"] & sf.ADVANCE else 0
    g = torch.Generator().manual_seed(3)
    start[B] = (torch.rand(BUILT, generator=g) * 0.5 * L).float()
    prog[PROG1], prog[PROG2], prog[PROG3], prog[PROG4] = 1 - adv, 2 - adv, 3 - adv, 4 - adv
    pd = lambda r: (torch.tensor([int(prog[r]) + adv]).float() * dt32)
    start[AT_LEN] = _time_at(float(L), pd(AT_LEN))
    start[BELOW_LEN] = _time_at(float(torch.nextafter(L, torch.tensor(0.0))), pd(BELOW_LEN))
    prog[ON_FRAME] = -adv
    start[ON_FRAME] = float(7 * mdt)
    start[PAST_END] = float(L) + 0.5
    start[CYC_PASS] = float(L) + 0.5
    cyc[CYC_PASS] = cyc[CYC_HOLD] = 3
    start[ONE_FRAME] = 0.013
    start[TWO_FRAMES] = float(0.37 * tb.dt[0])
    t_rew = sf.motion_time32(prog[B] + adv, cfg.dt, start[B], off[B])
    # on-pose bodies at t_rew, offsets chosen so that each threshold row's body lands at x ~ 0.6
    body[B] = _pose(tb, ids[B], t_rew, goff[B])
    q = body[B, :, 3:7]
    body[FLIPPED, :, 3:7] = -q[FLIPPED]
    half = lambda a, ax: torch.cat([torch.tensor(ax) * math.sin(a / 2), torch.tensor([math.cos(a / 2)])]).float()
    body[NEAR_PI, :, 3:7] = torch.nn.functional.normalize(qmul8_32(q[NEAR_PI], half(math.pi - 1e-3, [0.6, 0.8, 0.0]).expand(24, 4)), dim=-1)
    body[AT_PI, :, 3:7] = qmul8_32(q[AT_PI], torch.tensor([1.0, 0.0, 0.0, 0.0]).expand(24, 4))
    body[VERTICAL, 0, 3:7] = torch.tensor([0.5, 0.5, -0.5, 0.5])
    for r in (PROG1, PROG2, CYC_HOLD, RECOVERING):
        body[r, 5, 0:3] += 1.0                                    # a masked body far off its reference: fallen
    body[UNMASKED_FAR, 3, 0:3] += 1.0                             # body 3 is not a reset body
    _threshold_rows(tb, inp, cfg)


def _threshold_rows(tb, inp, cfg):
    """AT_TERM: one masked body exactly termination_distances[j] from its reference in the kernel's pinned fp32 order (not fallen);
    PAST_TERM: the same body one ulp farther (fallen).  The body and the time are chosen so that both forms a contracted lerp can take,
    fma(b, p1, (1 - b) p0) and fma(1 - b, p0, b p1), differ from the pinned one after the offset add, so an FMA in the reset position
    flips one of the two rows whichever product the compiler fuses."""
    ids, goff, body, start = inp["motion_ids"], inp["goff"], inp["body"], inp["start"]
    mid = ids[AT_TERM:AT_TERM + 1]
    term = inp["term"].float()
    adv = 1 if inp["flags"] & sf.ADVANCE else 0
    for k in range(64):
        st = start[AT_TERM:AT_TERM + 1] + 0.0123 * k
        t = sf.motion_time32(inp["progress"][AT_TERM:AT_TERM + 1] + adv, cfg.dt, st, inp["offset"][AT_TERM:AT_TERM + 1])
        i0, i1, b = po.frame_blend(t, tb.lengths[mid], tb.num_frames[mid], tb.dt[mid])
        s = tb.length_starts[mid[0]]
        p0, p1, bb = tb.gts[s + i0[0]], tb.gts[s + i1[0]], b[0]
        for j in [j for j in range(1, 24) if (inp["mask"] >> j) & 1]:
            lx = sf.lerp_rn32(p0[j, 0], p1[j, 0], bb)
            gx = torch.tensor(0.6, dtype=torch.float32) - lx
            forms = [contract32(p0[j, 0].reshape(1), p1[j, 0].reshape(1), bb.reshape(1), other)[0] + gx for other in (False, True)]
            if all(lx + gx != c for c in forms) and float(term[j]) < 0.6:
                for r in (AT_TERM, PAST_TERM):
                    start[r] = st[0]
                    goff[r] = torch.stack([gx, torch.tensor(0.0), torch.tensor(0.0)])
                    rp = sf.lerp_rn32(p0, p1, bb) + goff[r]
                    body[r, :, 0:3] = rp
                    body[r, j, 0] = rp[j, 0] - term[j]
                body[PAST_TERM, j, 0] = torch.nextafter(body[PAST_TERM, j, 0], torch.tensor(-math.inf))
                return j
    raise AssertionError("no body's contracted lerp differs from the pinned one")


def contract32(p0, p1, b, other=False):
    """The lerp with one product fused: fma(b, p1, (1 - b) p0), or (other) fma(1 - b, p0, b p1)."""
    return sf.fma32((1.0 - b).expand_as(p0), p0, b * p1) if other else sf.fma32(b.expand_as(p1), p1, (1.0 - b) * p0)


def built_mask(n: int) -> torch.Tensor:
    m = torch.zeros(n, dtype=torch.bool)
    m[:min(n, BUILT)] = True
    return m


# ---------------------------------------------------------------------------------------------------------------- fp32 simulations
def quat_angle32(q, wrap=True):
    w = q[..., 3]
    s = torch.sqrt(1.0 - w * w)
    ang = 2.0 * torch.acos(w)
    if wrap:
        ang = torch.where(ang >= sf.mf.PI32, ang - sf.mf.TWO_PI32, ang)
    return torch.where(s.abs() > 1e-5, ang, torch.zeros_like(ang))


def frame_blend32(t, length, nf, mdt):
    """frame_blend_rn: fminf / fmaxf take a NaN phase (0 / 0, a one-frame clip at time 0) to 0."""
    phase = t / length
    phase = torch.where(torch.isnan(phase), torch.zeros_like(phase), phase.clamp(0.0, 1.0))
    t = torch.where(t < 0, torch.zeros_like(t), t)
    i0 = (phase * (nf - 1).float()).long()
    i1 = torch.minimum(i0 + 1, nf - 1)
    return i0, i1, ((t - i0.float() * mdt) / mdt).clamp(0.0, 1.0)


def conj32(q):
    return torch.cat([-q[..., :3], q[..., 3:]], -1)


def sim_im_step(tb, inp, cfg, mut=None):
    """im_step_kernel in float32 on every env of inp: the outputs check_im_step reads, the full 934-float row."""
    flags = inp["flags"]
    do_rew, do_reset, do_obs = flags & 1, flags & 2, flags & 4
    body = inp["body"].float()[:, :24]
    n = body.shape[0]
    ids = inp["motion_ids"]
    adv = 1 if flags & sf.ADVANCE else 0
    prog = inp["progress"] + adv
    rec = (inp["recovery"] > 0) if (do_reset and inp["recovery"] is not None) else torch.zeros(n, dtype=torch.bool)
    rec_t = torch.zeros_like(rec) if mut == "no_pullback" else rec
    t_rew = sf.motion_time32(prog, cfg.dt, inp["start"], inp["offset"])
    t_obs = sf.motion_time32(prog + 1 - rec_t.long(), cfg.dt, inp["start"], inp["offset"])
    st = tb.length_starts[ids]

    def rows(t):
        i0, i1, b = frame_blend32(t, tb.lengths[ids], tb.num_frames[ids], tb.dt[ids])
        if mut == "i1_unclamped":
            i1 = i0 + 1
        return i0 + st, i1 + st, b

    f0r, f1r, b_rew = rows(t_rew)
    f0o, f1o, b_obs = rows(t_obs)
    if mut == "direct_slot2":                 # the fourth distinct row (obs f1) read from copy slot 2 (obs f0)
        four = (f0o != f0r) & (f0o != f1r) & (f1o != f0r) & (f1o != f1r) & (f0o != f1o) & (f0r != f1r)
        f1o = torch.where(four, f0o, f1o)
    goff = inp["goff"].float()[:, None, :]

    def pose(f0, f1, b, contract=None):
        bb = b[:, None, None]
        if contract is not None:
            p = contract32(tb.gts[f0], tb.gts[f1], bb, other=contract) + goff
        else:
            p = sf.lerp_rn32(tb.gts[f0], tb.gts[f1], bb) + goff
        return SimpleNamespace(p=p, q=slerp32(tb.grs[f0], tb.grs[f1], bb), v=(1.0 - bb) * tb.gvs[f0] + bb * tb.gvs[f1],
                               w=(1.0 - bb) * tb.gavs[f0] + bb * tb.gavs[f1])

    p, q, v, w = body[..., 0:3], body[..., 3:7], body[..., 7:10], body[..., 10:13]
    out = {"pass_time": (t_rew >= tb.lengths[ids]).to(torch.uint8)}
    progress = inp["progress"].clone()
    if adv:
        progress = torch.where(rec, progress, prog)
    if mut != "no_pullback":
        progress = torch.where(rec, prog - 1, progress)
    out["progress"] = progress
    r = pose(*((f0o, f1o, b_obs) if mut == "rew_at_obs" else (f0r, f1r, b_rew)), contract={"lerp_fma": False, "lerp_fma_other": True}.get(mut))
    if do_rew:
        sp = cfg.reward_specs
        e_pos = ((r.p - p) ** 2).sum(-1).sum(-1) * torch.tensor(1.0 / 72, dtype=torch.float32)
        th = quat_angle32(qmul8_32(r.q, conj32(q)), wrap=mut != "no_wrap")
        e_rot = (th * th).sum(-1) * torch.tensor(1.0 / 24, dtype=torch.float32)
        e_vel = ((r.v - v) ** 2).sum(-1).sum(-1) * torch.tensor(1.0 / 72, dtype=torch.float32)
        e_ang = ((r.w - w) ** 2).sum(-1).sum(-1) * torch.tensor(1.0 / 72, dtype=torch.float32)
        f = lambda k: torch.tensor(float(sp[k]), dtype=torch.float32)
        raw = [torch.exp(-f("k_pos") * e_pos), torch.exp(-f("k_rot") * e_rot), torch.exp(-f("k_vel") * e_vel), torch.exp(-f("k_ang_vel") * e_ang)]
        rew = f("w_pos") * raw[0] + f("w_rot") * raw[1] + f("w_vel") * raw[2] + f("w_ang_vel") * raw[3]
        if inp["dof_force"] is not None:
            pw = (inp["dof_force"] * inp["dof_vel"]).abs().sum(-1)
            p_rew = -torch.tensor(cfg.power_coefficient, dtype=torch.float32) * pw
            if mut != "power_early":
                p_rew = torch.where(prog <= 3, torch.zeros_like(p_rew), p_rew)
            raw.append(p_rew)
            rew = rew + p_rew
        out["raw"], out["rew"] = torch.stack(raw, 1), rew
    if do_reset:
        d = p - r.p
        x, y, z = d.unbind(-1)
        dist = torch.sqrt(sf.fma32(z, z, sf.fma32(y, y, x * x)))
        bits = torch.tensor([bool((inp["mask"] >> j) & 1) for j in range(24)])
        term = inp["term"].float()
        if cfg.use_mean_reset:
            s = torch.zeros(n)
            for j in range(24):
                s = s + torch.where(bits[j], dist[:, j], torch.zeros_like(s))
            cnt = 24.0 if mut == "mean_24" else float(bits.sum())
            first = int(torch.nonzero(bits)[0])
            fell = s / torch.tensor(cnt) > term[first]
        else:
            tj = term[0].expand(24) if mut == "term0" else term
            fell = ((dist > tj[None]) & bits[None]).any(-1)
        fell = fell & (prog > 1) & bool(cfg.enable_early_termination)
        pass_time = (prog >= cfg.max_episode_length - 1) if cfg.cycle_motion else (t_rew >= tb.lengths[ids])
        terminated = fell.long()
        reset = torch.where(pass_time, torch.ones_like(terminated), terminated)
        hold = (inp["cycle"] > 0) if mut == "cyc_always" else (~pass_time & (inp["cycle"] > 0))
        reset, terminated = torch.where(hold | rec, 0, reset), torch.where(hold | rec, 0, terminated)
        out.update(reset=reset, terminate=terminated, fdones=reset.float())
    if do_obs:
        r2 = pose(f0o, f1o, b_obs)
        root = body[:, 0:1]
        sb = body.clone()
        if mut == "heading_body1":
            sb[:, 0, 3:7] = body[:, 1, 3:7]
        h = heading_half32(sb[:, 0, 3:7])
        hb = h[:, None].expand(n, 24, 4)
        hf = hb * torch.tensor([1.0, 1.0, -1.0, 1.0])
        selfo = self_obs32(sb, True)
        dq = qmul8_32(hb, qmul8_32(r2.q, conj32(q)))
        if mut != "no_right":
            dq = qmul8_32(dq, hf)
        lp = r2.p - (p if mut == "lp_from_p" else root[..., 0:3])
        pieces = [qrot32(hb, r2.p - p), six32(dq), qrot32(hb, r2.v - v), qrot32(hb, r2.w - w), qrot32(hb, lp), six32(qmul8_32(hb, r2.q))]
        out["obs"] = torch.cat([selfo] + [x.reshape(n, -1) for x in pieces], 1)
        out["self_obs"] = selfo
        out.update(ref_body_pos=r2.p, ref_body_vel=r2.v, ref_body_rot=r2.q)
        a0, a1, ba = (f0r, f1r, b_rew) if mut == "dof_at_rew" else (f0o, f1o, b_obs)
        out["ref_dof_pos"] = expmap32(slerp32(tb.lrs[a0][:, 1:], tb.lrs[a1][:, 1:], ba[:, None, None])).reshape(n, 69)
    return out


def sim_task_obs(version, T, track_ids, upright, body, rp, rq, rv, rw, dof_pos=None, ref_dof=None, mut=None):
    """task_obs_kernel in float32: [n, size] rows in the kernel's own offsets (task_obs.cu)."""
    n, J = body.shape[0], len(track_ids)
    ids = torch.as_tensor(list(track_ids))
    h = heading_half32(base_removed32(body[:, 0, 3:7], upright))
    hb = h[:, None, None].expand(n, T, J, 4)
    hf = hb * torch.tensor([1.0, 1.0, -1.0, 1.0])
    sel = lambda x: x[:, None, ids].expand(n, T, J, x.shape[-1])
    p, q, v, w = sel(body[..., 0:3]), sel(body[..., 3:7]), sel(body[..., 7:10]), sel(body[..., 10:13])
    g = lambda x, c: x.reshape(n, T, 24, c)[:, :, ids]
    RP, RQ, RV, RW = g(rp, 3), g(rq, 4), g(rv, 3), g(rw, 3)
    d_pos = qrot32(hb, RP - p)
    d_rot = six32(qmul8_32(qmul8_32(hb, qmul8_32(RQ, conj32(q))), hf))
    d_vel, d_ang = qrot32(hb, RV - v), qrot32(hb, RW - w)
    l_pos, l_rot = qrot32(hb, RP - body[:, None, None, 0, 0:3]), six32(qmul8_32(hb, RQ))
    size = sf.task_obs_size(version, J, T)
    o = torch.zeros(n, size)
    t = torch.arange(T)[:, None].expand(T, J)
    j = torch.arange(J)[None, :].expand(T, J)
    if mut == "body_major":                   # item (t, j) stored where the layout puts item it = j T + t
        t, j = (j * T + t) // J, (j * T + t) % J
    it = t * J + j

    def put(base, width, val):
        cols = (base[..., None] + torch.arange(width)).reshape(-1)
        o[:, cols] = val.reshape(n, -1)

    if version == 7:
        ot = t * 9 * J
        put(ot + 3 * j, 3, d_pos), put(ot + 3 * J + 3 * j, 3, d_vel), put(ot + 6 * J + 3 * j, 3, l_pos)
    elif version in (1, 2, 3):
        put(3 * it, 3, d_pos), put(3 * T * J + 6 * it, 6, d_rot)
        if version != 3:
            put(9 * T * J + 3 * it, 3, d_vel), put(12 * T * J + 3 * it, 3, d_ang)
        if version == 2:
            b = ids[1:] if mut != "v2_track_index" else torch.arange(1, J)
            d0 = (3 * (b - 1))[:, None] + torch.arange(3)
            o[:, 15 * J:] = ref_dof[:, d0.reshape(-1)] - dof_pos[:, d0.reshape(-1)]
    elif version in (6, 8):
        ot = t * 24 * J
        put(ot + 3 * j, 3, d_pos), put(ot + 3 * J + 6 * j, 6, d_rot), put(ot + 9 * J + 3 * j, 3, d_vel), put(ot + 12 * J + 3 * j, 3, d_ang)
        put(ot + 15 * J + 3 * j, 3, l_pos), put(ot + 18 * J + 6 * j, 6, l_rot)
        if version == 8:
            put(24 * J + 3 * j, 3, qrot32(hb, RV)), put(27 * J + 3 * j, 3, qrot32(hb, RW))
    else:
        ot = t * (18 * J + 6)
        put(ot + 3 * j, 3, d_pos), put(ot + 3 * J + 6 * j, 6, d_rot)
        if mut == "v9_skeleton_root":             # body 0 of the skeleton instead of tracked body 0
            rv0, v0 = rv.reshape(n, T, 24, 3)[:, :, 0], body[:, None, 0, 7:10]
            rw0, w0 = rw.reshape(n, T, 24, 3)[:, :, 0], body[:, None, 0, 10:13]
        else:
            rv0, v0, rw0, w0 = RV[:, :, 0], v[:, :, 0], RW[:, :, 0], w[:, :, 0]
        put(ot[:, 0] + 9 * J, 3, qrot32(hb[:, :, 0], rv0 - v0)), put(ot[:, 0] + 9 * J + 3, 3, qrot32(hb[:, :, 0], rw0 - w0))
        put(ot + 9 * J + 6 + 3 * j, 3, l_pos), put(ot + 12 * J + 6 + 6 * j, 6, l_rot)
    return o


def task_obs_inputs(n: int, T: int, seed: int):
    """Random body states and fp32 reference arrays [n T, 24, .] (row e T + t); rows 0 and 1: a vertical and a w < 0 root."""
    g = torch.Generator().manual_seed(seed)
    unit = lambda *s: torch.nn.functional.normalize(torch.randn(*s, generator=g), dim=-1)
    body = torch.zeros(n, 24, 13)
    body[..., 0:3] = torch.randn(n, 24, 3, generator=g) * 0.4 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = unit(n, 24, 4)
    body[..., 7:13] = torch.randn(n, 24, 6, generator=g)
    body[0, 0, 3:7] = torch.tensor([0.5, 0.5, -0.5, 0.5])
    body[1, 0, 3:7] = -body[1, 0, 3:7].abs()
    rp = body[:, None, :, 0:3].expand(n, T, 24, 3).reshape(n * T, 24, 3) + 0.1 * torch.randn(n * T, 24, 3, generator=g)
    rq = unit(n * T, 24, 4)
    rv, rw = torch.randn(n * T, 24, 3, generator=g), torch.randn(n * T, 24, 3, generator=g)
    dof, rdof = torch.randn(n, 69, generator=g), torch.randn(n, 69, generator=g)
    return body, rp, rq, rv, rw, dof, rdof


TASK_CASES = [(1, 2, (0, 3, 5, 9, 13)), (2, 1, tuple(range(24))), (2, 1, (2, 5, 9, 17, 20)), (3, 3, (4,)), (1, 1, (0, 1, 2, 12, 22)), (1, 3, (7, 2, 19)), (6, 1, tuple(range(24))),
              (6, 3, (1, 6, 11, 18, 23)), (7, 3, (13, 18, 23)), (8, 1, (2, 5, 9, 17, 20)), (9, 3, (4, 8, 13, 18, 23)), (9, 1, (0,))]


# ---------------------------------------------------------------------------------------------------------------- tests
def _run(mut=None, fps=30.0, flags=7, recovery=True, power=True, **kw):
    cfg = config(**kw)
    tb = im_tables(40, seed=4, fps=fps)
    inp = im_inputs(tb, 257, seed=3, cfg=cfg, flags=flags, power=power, recovery=recovery)
    ref = sf.im_step_ref(table_dict(tb), inp, cfg)
    return inp, ref, sim_im_step(tb, inp, cfg, mut=mut)


VARIANTS = {"default": {}, "mixed rates": dict(fps=MIXED_RATES), "advance": dict(flags=7 | sf.ADVANCE),
            "no power": dict(power=False), "cycle": dict(cycle_motion=True, max_episode_length=30),
            "no early termination": dict(enable_early_termination=False),
            "mean reset": dict(use_mean_reset=True, mask=mask_of(DEFAULT_RESET_BODIES[1:]), term=nonuniform_term()),
            "per-body distances": dict(term=nonuniform_term()), "reward only": dict(flags=1), "reset obs": dict(flags=6),
            "obs only": dict(flags=4)}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_simulation_passes_every_link(variant):
    inp, ref, got = _run(**VARIANTS[variant])
    rep = sf.Report(f"im step {variant}")
    sf.check_im_step(rep, "im", got, ref, inp["flags"], built=built_mask(257))
    if inp["flags"] & sf.OBS:
        for track in ((6, (13, 2, 7)), (7, (23, 0, 5, 18)), (6, tuple(range(24))[::-1])):
            from pulse_b200.humanoid_im import track_columns
            tg = dict(got, obs=torch.cat([got["obs"][:, :358], got["obs"][:, 358:][:, track_columns(*track)]], 1))
            sf.check_im_step(rep, "im tracked", tg, ref, sf.OBS, track=track, built=built_mask(257))
    assert all(r[1] < 1.0 for r in rep.rows)
    if variant == "mixed rates":
        assert ref["four"] > 0


def test_built_edges_are_decided():
    """The threshold rows sit exactly on / one ulp past termination_distances[j] in the pinned order, both decided from the restatement;
    t_rew is exactly the clip length / one ulp below it; the fallen rows at progress 1 and 2 split on progress > 1."""
    inp, ref, got = _run()
    d32 = ref["dist"][0]
    term = inp["term"]
    assert bool((d32[AT_TERM] == term).any()) and bool(((d32[PAST_TERM] > term) & (d32[PAST_TERM] == torch.nextafter(term, torch.tensor(1.0)))).any())
    assert ref["terminate"][[AT_TERM, PAST_TERM, UNMASKED_FAR, PROG1, PROG2]].tolist() == [0, 1, 0, 0, 1]
    assert ref["pass_time"][[AT_LEN, BELOW_LEN]].tolist() == [1, 0]
    assert ref["reset"][[CYC_PASS, CYC_HOLD, RECOVERING]].tolist() == [1, 0, 0]
    assert float(ref["raw"][0][0][ON_POSE]) > 0.999 and float(ref["raw"][4][0][PROG3]) == 0.0 and float(ref["raw"][4][0][PROG4]) < 0.0


MUTATIONS = [
    ("rew_at_obs", {}, "reward raw pos"),
    ("i1_unclamped", {}, "reward raw pos"),
    ("direct_slot2", dict(fps=MIXED_RATES), "task dp"),
    ("lerp_fma", {}, "terminate"),
    ("lerp_fma_other", {}, "terminate"),
    ("lerp_fma", dict(fps=MIXED_RATES), "terminate"),
    ("lerp_fma_other", dict(fps=MIXED_RATES, term=nonuniform_term()), "terminate"),
    ("no_wrap", {}, "reward raw rot"),
    ("power_early", {}, "reward raw power"),
    ("mean_24", dict(use_mean_reset=True, mask=mask_of(DEFAULT_RESET_BODIES[1:]), term=nonuniform_term()), "terminate (fp64 decided)"),
    ("term0", dict(term=nonuniform_term()), "terminate (fp64 decided)"),
    ("cyc_always", {}, "reset"),
    ("no_pullback", {}, "progress"),
    ("heading_body1", {}, "self body pos"),
    ("no_right", {}, "task drot"),
    ("lp_from_p", {}, "task lp"),
    ("dof_at_rew", {}, "ref dof pos"),
]


@pytest.mark.parametrize("mut,kw,link", MUTATIONS, ids=[m[0] + ("-" + "-".join(m[1]) if m[1] else "") for m in MUTATIONS])
def test_mutation_fails_its_link(mut, kw, link):
    inp, ref, got = _run(mut=mut, **kw)
    with pytest.raises(sf.BoundError, match=f"^im {re.escape(link)}:"):
        sf.check_im_step(None, "im", got, ref, inp["flags"], built=built_mask(257))


@pytest.mark.parametrize("upright", [True, False])
@pytest.mark.parametrize("case", TASK_CASES, ids=[f"v{c[0]}-T{c[1]}-J{len(c[2])}" for c in TASK_CASES])
def test_task_obs_simulation_passes_every_link(case, upright):
    version, T, ids = case
    args = task_obs_inputs(97, T, seed=version)
    ref = sf.task_obs_ref(version, T, ids, upright, *args)
    rep = sf.Report(f"task obs v{version}")
    sf.check_task_obs(rep, "task", sim_task_obs(version, T, ids, upright, *args), ref, built=torch.arange(97) < 2)
    assert all(r[1] < 1.0 for r in rep.rows)


TASK_MUTATIONS = [("v9_skeleton_root", (9, 3, (4, 8, 13, 18, 23)), "root dv"), ("v2_track_index", (2, 1, (2, 5, 9, 17, 20)), "dof"),
                  ("body_major", (1, 3, (0, 3, 5, 9, 13)), "dp"), ("body_major", (6, 3, (1, 6, 11, 18, 23)), "dp")]


@pytest.mark.parametrize("mut,case,link", TASK_MUTATIONS, ids=[f"{m[0]}-v{m[1][0]}" for m in TASK_MUTATIONS])
def test_task_obs_mutation_fails_its_link(mut, case, link):
    version, T, ids = case
    args = task_obs_inputs(97, T, seed=version)
    ref = sf.task_obs_ref(version, T, ids, True, *args)
    with pytest.raises(sf.BoundError, match=f"^task {link}:"):
        sf.check_task_obs(None, "task", sim_task_obs(version, T, ids, True, *args, mut=mut), ref)


def test_fma32_rounds_once():
    """fma32 against exact rational arithmetic, halfway cases included."""
    from fractions import Fraction
    g = torch.Generator().manual_seed(1)
    a, b, c = (torch.randn(4000, generator=g) for _ in range(3))
    a[:1000] = 1.0 + torch.randint(0, 1 << 12, (1000,), generator=g).float() * 2.0 ** -23
    b[:1000] = 1.0 + 2.0 ** -12
    c[:1000] = -1.0
    got = sf.fma32(a, b, c)
    for k in range(0, 4000, 7):
        exact = Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k]))
        lo = torch.tensor(float(exact), dtype=torch.float32)
        cands = [lo, torch.nextafter(lo, torch.tensor(math.inf)), torch.nextafter(lo, torch.tensor(-math.inf))]
        best = min(cands, key=lambda x: (abs(Fraction(float(x)) - exact), int(x.view(torch.int32)) & 1))
        assert float(got[k]) == float(best), k
