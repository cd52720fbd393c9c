"""The reset kernels' float64 references (tests/reset_fp64.py) have teeth: a CPU simulation of each kernel passes every link, and a
simulation with one defect fails the link it breaks with BoundError naming it.  The simulations restate the arithmetic of
reset_warps.cuh, ztask_reset.cu, terrain_reset.cu, terrain.cu (traj_generate) and humanoid_obs.cuh in float32 torch operations, and the
integer work of getup_reset.cu env by env and state by state."""
import math

import numpy as np
import pytest
import torch

from oracle import pulse_oracle as po
from tests import reset_fp64 as rf
from tests.helpers import exact_tables
from tests.test_motion_fp64_cpu import expmap32, qmul8_32, slerp32

RATES = [24.0, 25.0, 29.97, 30.0, 50.0, 60.0, 120.0]
KEYS = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "lengths", "num_frames", "dt", "length_starts")
SEED, OFF = 77, 5
STRIKE = dict(near_prob=0.5, near_dist=1.5, dmin=0.5, dmax=10.0)
TASK = dict(dist_max=1.0, height_min=0.5, height_max=1.5, speed_min=0.0, speed_max=5.0)
DT = float(np.float32(1.0 / 60.0) * 2)
HSCALE, VSCALE = 0.1, 0.005


# ---------------------------------------------------------------------------------------------------------------- fp32 pieces
def qrot32(q, v):
    s = 2.0 * q[..., 3:] ** 2 - 1.0
    d = 2.0 * (q[..., :3] * v).sum(-1, keepdim=True)
    return v * s + torch.cross(q[..., :3], v, dim=-1) * (2.0 * q[..., 3:]) + q[..., :3] * d


def base_removed32(q, upright):
    return q if upright else qmul8_32(q, torch.tensor(rf.BASE_INV).expand_as(q))


def heading_inv32(q):
    """heading_half: (0, 0, -hs, hc)."""
    x, y, z, w = q.unbind(-1)
    s = 2.0 * w * w - 1.0
    rx, ry = s + 2.0 * x * x, 2.0 * w * z + 2.0 * x * y
    inv = torch.rsqrt(rx * rx + ry * ry)
    ch, sh = rx * inv, ry * inv
    pos = ch >= 0
    c1 = torch.sqrt(0.5 * (1.0 + ch))
    s2 = torch.copysign(torch.sqrt(0.5 * (1.0 - ch)), sh)
    hc = torch.where(pos, c1, 0.5 * sh / s2)
    hs = torch.where(pos, 0.5 * sh / c1, s2)
    return torch.stack([torch.zeros_like(hs), torch.zeros_like(hs), -hs, hc], -1)


def six32(q):
    x, y, z, w = q.unbind(-1)
    s = 2.0 * w * w - 1.0
    return torch.stack([s + x * 2 * x, z * 2 * w + y * 2 * x, -y * 2 * w + z * 2 * x, y * 2 * w + x * 2 * z, -x * 2 * w + y * 2 * z,
                        s + z * 2 * z], -1)


def exp_map_quat32(e, branch=True):
    ang = e.norm(dim=-1, keepdim=True)
    axis = e / ang
    ang = torch.atan2(torch.sin(ang), torch.cos(ang))
    if branch:
        small = ~(ang.abs() > 1e-5)
        ang = torch.where(small, torch.zeros_like(ang), ang)
        axis = torch.where(small, torch.tensor([0.0, 0.0, 1.0]).expand_as(axis), axis)
    q = torch.cat([axis * torch.sin(0.5 * ang), torch.cos(0.5 * ang)], -1)
    return q / q.norm(dim=-1, keepdim=True)


def amp_row32(p0, q0, v0, w0, dof, dvel, key, width, upright, mut=None):
    """store_amp_row: [h | six(hinv q0) | R v0 | R w0 | 19 six(dof) | 57 dof vel | 4 R(key - p0)] of base_rot_removed(q0)."""
    qb = base_removed32(q0, upright)
    h = heading_inv32(qb)
    rot = lambda v: qrot32(h.reshape(h.shape[:1] + (1,) * (v.dim() - 2) + (4,)).expand(v.shape[:-1] + (4,)), v)
    kj = torch.tensor(rf.KEPT_JOINTS)
    d = dof.reshape(len(p0), 23, 3)[:, kj]
    rel = key - p0[:, None]
    row = torch.cat([p0[:, 2:3], six32(qmul8_32(h, qb)), rot(v0), rot(w0), six32(exp_map_quat32(d, branch=mut != "no_small_angle")).reshape(len(p0), -1),
                     dvel.reshape(len(p0), 23, 3)[:, kj].reshape(len(p0), -1), (rel if mut == "key_world" else rot(rel)).reshape(len(p0), -1)], 1)
    skip = 196 - width
    if mut == "shift_195" and width == 195:
        skip = 0
    return row[:, skip:skip + width]


def gather32(t, mids, times):
    i0, i1, b = po.frame_blend(times, t["lengths"][mids], t["num_frames"][mids], t["dt"][mids])
    f0, f1 = i0 + t["length_starts"][mids], i1 + t["length_starts"][mids]
    bb = b[:, None, None]
    lerp = lambda k: (1.0 - bb) * t[k][f0] + bb * t[k][f1]
    return {"f0": f0, "f1": f1, "pos": lerp("gts"), "vel": lerp("gvs"), "ang": lerp("gavs"), "rot": slerp32(t["grs"][f0], t["grs"][f1], bb),
            "dof": expmap32(slerp32(t["lrs"][f0][:, 1:], t["lrs"][f1][:, 1:], bb)).reshape(len(mids), -1),
            "dvel": ((1.0 - b[:, None]) * t["dvs"][f0].reshape(len(mids), -1) + b[:, None] * t["dvs"][f1].reshape(len(mids), -1))}


# ---------------------------------------------------------------------------------------------------------------- the reset kernels
def sim_reset(t, cdf, floor, envs, pose, upright, strike=False, width=196, steps=3, terrain=None, mut=None):
    """ztask_reset_kernel / terrain_reset_kernel over the env list `envs` with Philox draws (SEED, OFF)."""
    e = envs.numpy().astype(np.uint64)
    r0 = rf.words(SEED, e, OFF)
    wx, wy = (1, 0) if mut == "swap_phase_clip" else (0, 1)
    ph, mu = rf.uniform(r0[:, wx]), rf.uniform(r0[:, wy])
    mids = rf.pick_motion_ref(cdf, mu)
    t0 = rf.start_time_ref(ph, t["lengths"][mids])
    g = gather32(t, mids, t0)
    pos = g["pos"].clone()
    fl = floor[g["f1"] if mut == "floor_f1" else g["f0"]]
    d = (fl + pos[:, 0, 2]) - 0.02
    pos[..., 2] = pos[..., 2] - d[:, None]
    rot, vel, ang = g["rot"].clone(), g["vel"].clone(), g["ang"].clone()
    rp = pos[:, 0].clone()
    root = torch.cat([rp, rot[:, 0], vel[:, 0], ang[:, 0]], 1)
    out = {"mids": mids, "t0": t0}
    if pose == rf.POSE_FACE_X:
        h = heading_inv32(base_removed32(rot[:, 0], upright))
        hb = h[:, None].expand(rot.shape)
        pos = qrot32(hb, pos - rp[:, None]) + rp[:, None]
        rot, vel = qmul8_32(hb, rot), qrot32(hb, vel)
        root = torch.cat([rp, rot[:, 0], vel[:, 0], qrot32(h, ang[:, 0])], 1)
    elif pose == rf.POSE_ROOT_XY_ZERO:
        root[:, :2] = 0.0
    if terrain is not None:
        hf, cx, cy, pts = terrain
        word = r0[:, 3] if mut == "loc_from_w" else r0[:, 2]
        loc = ((word.numpy().astype(np.uint64) * np.uint64(len(cx))) >> np.uint64(32)).astype(np.int64)
        loc = torch.from_numpy(loc)
        nx, ny = cx[loc], cy[loc]
        dx, dy = nx - root[:, 0], ny - root[:, 1]
        old = root[:, :2].clone()
        root[:, 0], root[:, 1] = nx, ny
        at = old if mut == "center_old_xy" else root[:, :2]
        root[:, 2] = root[:, 2] + center_height32(hf, pts, root[:, 3:7], at, upright)
        if mut == "lift_bodies":
            pos[..., 2] = pos[..., 2] + center_height32(hf, pts, root[:, 3:7], root[:, :2], upright)[:, None]
        pos[..., 0] = pos[..., 0] + dx[:, None]
        pos[..., 1] = pos[..., 1] + dy[:, None]
        out["loc"] = loc
    body = torch.cat([pos, rot, vel, ang], -1)
    out.update(body=body, root=root, dof_pos=g["dof"], dof_vel=g["dvel"])
    if strike:
        r1 = rf.words(SEED, e if mut == "strike_no_stream" else e + np.uint64(rf.STRIKE_STREAM), OFF)
        u = torch.stack([rf.uniform(r0[:, 2]), rf.uniform(r0[:, 3]), rf.uniform(r1[:, 0]), rf.uniform(r1[:, 1])], 1)
        dm = torch.where(u[:, 0] < STRIKE["near_prob"], torch.tensor(STRIKE["near_dist"]), torch.tensor(STRIKE["dmax"]))
        dist = (dm - STRIKE["dmin"]) * u[:, 1] + STRIKE["dmin"]
        th, yaw = TWO_PI * u[:, 2], TWO_PI * u[:, 3]
        out["target"] = torch.stack([dist * torch.cos(th) + root[:, 0], dist * torch.sin(th) + root[:, 1], torch.sin(0.5 * yaw),
                                     torch.cos(0.5 * yaw)], 1)
    kb = torch.tensor(rf.KEY_BODIES)
    rows = [amp_row32(body[:, 0, 0:3], body[:, 0, 3:7], body[:, 0, 7:10], body[:, 0, 10:13], out["dof_pos"], out["dof_vel"], body[:, kb, 0:3],
                      width, upright, mut)]
    times = rf.history_times(t0, DT, steps)
    for k in range(1, steps):
        gk = gather32(t, mids, times[:, k])
        p = gk["pos"].clone()
        if mut == "fix_history":
            fk = floor[gk["f0"]]
            p[..., 2] = p[..., 2] - ((fk + p[:, 0, 2]) - 0.02)[:, None]
        rows.append(amp_row32(p[:, 0], gk["rot"][:, 0], gk["vel"][:, 0], gk["ang"][:, 0], gk["dof"], gk["dvel"], p[:, kb], width, upright, mut))
    out["amp"] = torch.stack(rows, 1)
    return out


TWO_PI = torch.tensor(rf.TWO_PI32)


def center_height32(hf, pts, rr, xy, upright):
    qb = base_removed32(rr, upright)
    n = torch.sqrt(qb[:, 2] ** 2 + qb[:, 3] ** 2).clamp_min(1e-9)
    qy = torch.stack([torch.zeros_like(n), torch.zeros_like(n), qb[:, 2] / n, qb[:, 3] / n], -1)
    P = pts.shape[0]
    q = qy[:, None].expand(-1, P, 4)
    u = q[..., :3]
    b = pts[None].expand(len(rr), P, 3)
    tt = torch.cross(u, b, dim=-1) * 2.0
    r = b + q[..., 3:] * tt + torch.cross(u, tt, dim=-1)
    x, y = r[..., 0] + xy[:, None, 0], r[..., 1] + xy[:, None, 1]
    px = (x / HSCALE).long().clamp(0, hf.shape[0] - 2)
    py = (y / HSCALE).long().clamp(0, hf.shape[1] - 2)
    h = torch.minimum(hf[px, py].long(), hf[px + 1, py + 1].long()).float() * VSCALE
    return h.sum(-1) / P


def sim_task(envs, progress, kind, mut=None):
    r = rf.words(SEED, envs.numpy().astype(np.uint64) + np.uint64(rf.TASK_STREAM), OFF)
    shift = 31 if mut == "steps_31" else 32
    steps = 100 + ((r[:, 3].numpy().astype(np.uint64) * np.uint64(100)) >> np.uint64(shift)).astype(np.int64)
    u = torch.stack([rf.uniform(r[:, c]) for c in range(3)], 1)
    if kind == "reach":
        tgt = torch.cat([TASK["dist_max"] * (2.0 * u[:, :2] - 1.0), (TASK["height_max"] - TASK["height_min"]) * u[:, 2:3] + TASK["height_min"]], 1)
    else:
        tgt = (TASK["speed_max"] - TASK["speed_min"]) * u[:, 0] + TASK["speed_min"]
    return tgt, progress + torch.from_numpy(steps)


# ---------------------------------------------------------------------------------------------------------------- fixtures
def _tables():
    tb = exact_tables(14, seed=4, fps=RATES)
    t = {k: getattr(tb, k).clone() for k in KEYS}
    s, nf = int(t["length_starts"][3]), int(t["num_frames"][3])
    t["lrs"][s:s + nf, 1:5] = torch.tensor([0.0, 0.0, 0.0, 1.0])     # identity joints: the exp-map zero and the 1e-5 identity branch
    return t


def _cdf(m):
    p = torch.rand(m, generator=torch.Generator().manual_seed(3))
    p[[2, 6]] = 0.0
    return torch.cumsum(p / p.sum(), 0)


def _floor(t):
    return -0.9 + 0.1 * torch.rand(t["gts"].shape[0], generator=torch.Generator().manual_seed(5))


def _terrain():
    g = torch.Generator().manual_seed(6)
    hf = torch.randint(-200, 200, (80, 90), generator=g, dtype=torch.int16)
    cells = torch.randint(5, 70, (300, 2), generator=g)
    cx, cy = (cells[:, 0].float() * HSCALE), (cells[:, 1].float() * HSCALE)
    from pulse_b200.terrain import center_height_points
    return hf, cx, cy, center_height_points().float()


def _check_reset(kind, upright=True, width=196, mut=None, n=900):
    t = _tables()
    M = t["lengths"].shape[0]
    cdf, floor = _cdf(M), _floor(t)
    envs = torch.arange(0, 3 * n, 3)
    pose = {"reach": rf.POSE_ROOT_XY_ZERO, "strike": rf.POSE_ROOT_XY_ZERO, "speed": rf.POSE_FACE_X, "terrain": rf.POSE_AS_IS}[kind]
    terrain = _terrain() if kind == "terrain" else None
    got = sim_reset(t, cdf, floor, envs, pose, upright, strike=kind == "strike", width=width, terrain=terrain, mut=mut)
    dr = rf.ztask_draws(SEED, envs, OFF)
    mids = rf.pick_motion_ref(cdf, dr["motion_u"])
    rf.check_exact(None, "draws clip", got["mids"], mids)
    t0 = rf.start_time_ref(dr["phase"], t["lengths"][mids])
    rf.check_exact(None, "draws start time", got["t0"], t0)
    ref = rf.reset_state_ref(t, mids, t0, floor, pose, upright)
    if kind == "terrain":
        hf, cx, cy, pts = terrain
        loc = rf.terrain_loc(dr["r0"], len(cx))
        rf.check_exact(None, "terrain location", got["loc"], loc)
        sp = rf.spawn_ref(ref, loc, cx, cy, hf, HSCALE, VSCALE, pts, upright, got["root"][:, 3:7])
        ref["body_pos"], ref["root_pos"] = sp["body_pos"], sp["root_pos"]
        rf.limit_share(None, "terrain cell edge", sp["edge"], amb_max=rf.EDGE_MAX)
    rf.check_state(None, kind, got, ref)
    if kind == "strike":
        s = rf.strike_ref(dr["strike_u"], torch.zeros(n, 2), STRIKE["near_prob"], STRIKE["near_dist"], STRIKE["dmin"], STRIKE["dmax"])
        rf.check(None, "strike target xy", got["target"][:, :2], *s["xy"])
        rf.check(None, "strike target yaw", got["target"][:, 2:], *s["zw"])
    if kind in ("reach", "speed"):
        prog = torch.randint(0, 50, (n,), generator=torch.Generator().manual_seed(2))
        tgt, chg = sim_task(envs, prog, kind, mut)
        td = rf.task_draws(SEED, envs, OFF, 100, 200)
        tr = rf.task_ref(kind, td["rand"], td["steps"], prog, **TASK)
        rf.check_exact(None, "task change steps", chg, tr["change_steps"])
        rf.check(None, "task target", tgt, *tr["target"])
    body = got["body"]
    rf.check_amp(None, "row 0", got["amp"][:, 0], rf.state_amp_ref(body, got["dof_pos"], got["dof_vel"], upright))
    times = rf.history_times(t0, DT, got["amp"].shape[1])
    for k in range(1, got["amp"].shape[1]):
        rf.check_amp(None, f"row {k}", got["amp"][:, k], rf.motion_amp_ref(rf.motion_ref(t, mids, times[:, k]), upright))


def sim_getup_kernels(envs, term, avail, assign, rec_u, fall_u, key_bits, p_rec, p_fall, steps, counter):
    """getup_classify / getup_keys / getup_select / getup_apply restated env by env and state by state: the release, the free count,
    the classification in ascending env order with a running fall slot, the 64-bit keys (bits << 32 | s, all ones when held), and the
    rank of each free key among all keys."""
    avail, assign, counter = avail.clone(), assign.clone(), counter.clone()
    for e in envs.tolist():
        avail[int(assign[e])] = 0
    free = int((avail == 0).sum())
    ref_l, fall_l, rec_l, slot = [], [], [], 0
    for e in envs.tolist():
        rec = bool(rec_u[e] < np.float32(p_rec)) and int(term[e]) == 1
        fall = not rec and bool(fall_u[e] < np.float32(p_fall))
        if fall:
            fall, slot = slot < free, slot + 1
        (rec_l if rec else fall_l if fall else ref_l).append(e)
        counter[e] = 0 if not rec and not fall else steps
    falls = min(slot, free)
    held = np.uint64(0xFFFFFFFFFFFFFFFF)
    keys = np.array([held if int(avail[s]) else (np.uint64(int(key_bits[s])) << np.uint64(32)) | np.uint64(s) for s in range(len(avail))],
                    dtype=np.uint64)
    rank = (keys[None, :] < keys[:, None]).sum(1)
    pick = [-1] * falls
    for s in range(len(avail)):
        if keys[s] != held and rank[s] < falls:
            pick[int(rank[s])] = s
    for e, st in zip(fall_l, pick):
        avail[st] = 1
        assign[e] = st
    L = lambda x: torch.tensor(x, dtype=torch.int64)
    return {"ref_list": L(ref_l), "fall_list": L(fall_l[:falls]), "recovery_list": L(rec_l), "fall_pick": L(pick),
            "class_counts": torch.tensor([len(ref_l), falls, len(rec_l)], dtype=torch.int32), "error": slot - falls, "avail": avail,
            "assign": assign, "counter": counter}


def sim_getup(n, P, mut=None, rec_frac=0.5):
    g = torch.Generator().manual_seed(12)
    envs = (torch.rand(n, generator=g) < 0.6).nonzero().flatten()
    term = (torch.rand(n, generator=g) < rec_frac).long()
    avail = (torch.rand(P, generator=g) < 0.5).long()
    assign = torch.randint(0, P, (n,), generator=g)
    counter = torch.randint(0, 9, (n,), generator=g, dtype=torch.int32)
    r = rf.words(SEED, envs.numpy().astype(np.uint64), OFF)
    kw = rf.words(SEED, np.arange(P, dtype=np.uint64), OFF)[:, 0 if mut == "keys_from_x" else 3]
    rec_u, fall_u = torch.ones(n), torch.ones(n)
    rec_u[envs], fall_u[envs] = rf.uniform(r[:, 1]), rf.uniform(r[:, 2])
    got = sim_getup_kernels(envs, term, avail, assign, rec_u, fall_u, kw, 0.3, 0.6, 60, counter)
    dr = rf.getup_draws(SEED, envs, OFF, P)
    ru, fu = torch.ones(n), torch.ones(n)
    ru[envs], fu[envs] = dr["recovery_u"], dr["fall_u"]
    want = rf.getup_ref(envs, term, avail, assign, ru, fu, dr["key_bits"], 0.3, 0.6, 60, counter)
    for k in ("ref_list", "fall_list", "recovery_list", "class_counts", "fall_pick", "avail", "assign", "counter"):
        rf.check_exact(None, f"getup {k}", got[k], want[k])
    rf.check_exact(None, "getup error", torch.tensor(got["error"]), torch.tensor(want["error"]))
    return want


TRAJ = dict(dtheta_scale=2.0 * 0.1, dspeed_scale=2.0 * 0.1, seg_dt=0.1, speed_min=0.0, speed_max=3.0, sharp_turn_prob=0.02)


def sim_traj(start, envs, mut=None):
    """traj_list_kernel (terrain.cu traj_generate) in float32, Philox blocks (SEED, e + 4 * 2^32, 101 * OFF + k)."""
    S = rf.TRAJ_SEGS
    stream = 0 if mut == "traj_no_stream" else rf.TRAJ_STREAM
    base = OFF if mut == "traj_counter" else rf.TRAJ_VERTS * OFF
    e = envs.numpy().astype(np.uint64) + np.uint64(stream)
    f = lambda x: torch.tensor(x, dtype=torch.float32)
    pi, p = f(3.14159265358979), f(TRAJ["sharp_turn_prob"])
    smin, smax, segdt = f(TRAJ["speed_min"]), f(TRAJ["speed_max"]), f(TRAJ["seg_dt"])
    hb = rf.words(SEED, e, base + S)
    u_head, u_v0 = rf.uniform(hb[:, 0]), rf.uniform(hb[:, 1])
    n = len(e)
    out = torch.zeros(n, rf.TRAJ_VERTS, 3)
    out[:, 0, :2] = start
    ang, px, py = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for k in range(S):
        b = rf.words(SEED, e, base + k)
        u = [rf.uniform(b[:, c]) for c in range(4)]
        if k == 0:
            dth = pi * (2.0 * u_head - 1.0)
            speed = (smax - smin) * u_v0 + smin
        else:
            dth = torch.where(u[2] < p, pi * (2.0 * u[1] - 1.0), (2.0 * u[0] - 1.0) * f(TRAJ["dtheta_scale"]))
            speed = torch.clamp(speed + (2.0 * u[3] - 1.0) * f(TRAJ["dspeed_scale"]), float(smin), float(smax))
        ang = ang + dth.double()
        th = ang.float()
        seg = speed * segdt
        dx, dy = torch.cos(th) * seg, -torch.sin(th) * seg
        if k == 0:
            dx, dy = dx + start[:, 0], dy + start[:, 1]
        px, py = px + dx.double(), py + dy.double()
        out[:, k + 1, 0], out[:, k + 1, 1] = px.float(), py.float()
    return out


def _check_traj(mut=None, n=700):
    envs = torch.arange(0, 5 * n, 5)
    start = (torch.rand(n, 2, generator=torch.Generator().manual_seed(9)) * 12.0).float()
    got = sim_traj(start, envs, mut)
    rf.check_traj(None, "trajectory", got, start, rf.traj_ref(start, rf.traj_draws(SEED, envs, OFF), **TRAJ))


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("kind,upright,width", [("reach", True, 195), ("speed", True, 196), ("speed", False, 195), ("strike", True, 196),
                                                ("terrain", True, 196), ("terrain", False, 195)])
def test_simulated_reset_passes_every_link(kind, upright, width):
    _check_reset(kind, upright, width)


@pytest.mark.parametrize("kind,mut,link,width", [
    ("reach", "swap_phase_clip", "draws clip", 196), ("strike", "strike_no_stream", "strike target xy", 196), ("reach", "steps_31", "task change steps", 196),
    ("terrain", "loc_from_w", "terrain location", 196), ("reach", "floor_f1", "body pos", 196), ("reach", "fix_history", "amp h", 196),
    ("reach", "key_world", "amp key", 195), ("speed", "no_small_angle", "amp dof six", 196), ("reach", "shift_195", "amp", 195),
    ("terrain", "lift_bodies", "body pos", 196), ("terrain", "center_old_xy", "root pos", 196)])
def test_reset_mutation_fails_its_link(kind, mut, link, width):
    with pytest.raises(rf.BoundError, match=link):
        _check_reset(kind, width=width, mut=mut)


def test_simulated_getup_passes_and_keys_from_x_fail():
    want = sim_getup(700, 300)
    assert int(want["class_counts"][1]) > 0 and int(want["class_counts"][2]) > 0
    exhausted = sim_getup(700, 40, rec_frac=0.1)                 # more fall envs than free states: the surplus takes reference episodes
    assert exhausted["error"] > 0
    with pytest.raises(rf.BoundError, match="getup fall_pick"):
        sim_getup(700, 300, mut="keys_from_x")


def test_exhausted_pool_surplus_takes_reference_episodes():
    """More fall envs than free states: the first `free` of them in env order fall, the rest take a reference-state episode, and the
    surplus is the error increment."""
    n, P = 64, 8
    envs = torch.arange(n)
    avail = torch.ones(P, dtype=torch.int64)
    assign = torch.zeros(n, dtype=torch.int64)
    assign[:] = 1
    assign[:3] = torch.tensor([1, 4, 6])
    r = rf.getup_ref(envs, torch.zeros(n, dtype=torch.int64), avail, assign, torch.ones(n), torch.zeros(n), torch.arange(P), 0.3, 0.5, 9,
                     torch.zeros(n, dtype=torch.int32))
    assert r["class_counts"].tolist() == [n - 3, 3, 0] and r["error"] == n - 3
    assert r["fall_list"].tolist() == [0, 1, 2] and r["fall_pick"].tolist() == [1, 4, 6]


def test_pick_motion_edges():
    """u = 1.0 gives u * total = total, which the nextafter clamp keeps below total: the pick is the last clip with weight, not the
    trailing zero-weight clip an unclamped search would reach.  The largest u01, one ulp below 1, stays below total by itself.  Zero-weight
    clips are never picked; u = 0 takes the first clip with weight."""
    cdf = torch.cumsum(torch.tensor([0.0, 0.25, 0.0, 0.5, 0.25, 0.0]), 0)
    u = torch.tensor([0.0, float(np.float32(1 - 2 ** -24)), 0.25, 0.2499999, 0.75, 1.0])
    assert rf.pick_motion_ref(cdf, u).tolist() == [1, 4, 3, 1, 4, 4]
    unclamped = int(torch.searchsorted(cdf, cdf[-1:], right=True).clamp(max=len(cdf) - 1))
    assert unclamped == 5                                  # what the search gives without the clamp: the zero-weight last clip


def test_simulated_trajectory_passes():
    _check_traj()


@pytest.mark.parametrize("mut", ["traj_no_stream", "traj_counter"])
def test_trajectory_mutation_fails_its_link(mut):
    """The stream without + 4 * 2^32, or the counter offset + k instead of 101 * offset + k, draws other waypoints."""
    with pytest.raises(rf.BoundError, match="traj verts"):
        _check_traj(mut)


def test_start_time_edges():
    """Phase 0 starts at 0; one ulp below 1 stays on the 1/30 grid inside the clip; a 2-frame clip's start is 0 or 1/30."""
    mlen = torch.tensor([1.0 / 30, 1.0 / 24, 2.5, 1.0 / 120], dtype=torch.float32)
    t0 = rf.start_time_ref(torch.zeros(4), mlen)
    assert not t0.any()
    t1 = rf.start_time_ref(torch.full((4,), float(np.float32(1 - 2 ** -24))), mlen)
    assert bool((t1 <= mlen).all()) and bool((t1 >= 0).all())
    assert math.isclose(float(t1[2]) * 30, round(float(t1[2]) * 30), abs_tol=1e-4)
