"""The task steps' float64 references (tests/step_fp64.py) have teeth: a float32 CPU simulation of each step kernel passes every link,
and a simulation with one defect fails the link it breaks with BoundError naming it.  The simulations restate the arithmetic of
ztask_env.cuh (ztask_env for the SMPL reach, SMPL speed / strike, SMPL-X speed and SMPL-X reach / strike layouts) and terrain.cu / terrain_height.cuh
(terrain_env, whose _rn intrinsics are the round-to-nearest float32 operations torch performs on the CPU) in float32 torch operations.
The input generators (with the built edge envs) are shared with tests/test_gpu_task_step_fp64.py."""
import math

import numpy as np
import pytest
import torch

from tests import step_fp64 as sf
from tests.test_motion_fp64_cpu import qmul8_32
from tests.test_reset_fp64_cpu import qrot32, six32

MAX_LEN = 300
DT = float(np.float32(1.0 / 30.0))
SMPLX_CONTACTS = (7, 3, 8, 4, 40, 47)            # feet and two bodies of the second slot
SMPLX_STRIKE = (35, 36, 45)
SMPL_CONTACTS = (7, 3, 8, 4)
SMPL_STRIKE = (18, 19, 20, 21, 22, 23)
REACH_IDS = {24: (23,), 52: (0, 31, 32, 51)}
# a target rotation whose 2 w^2 - 1 + 2 z^2 is 0.2f in fp32 in every contraction order: rot_err < 0.2 is false, exactly
ROT_EDGE = (0.0, 0.0, 0.15776729583740234, 0.7583597302436829)
BUILT = 16                                       # rows 0 .. BUILT - 1 of every generated batch are the built edge envs


def mask_of(ids) -> int:
    m = 0
    for j in ids:
        m |= 1 << j
    return m


# ---------------------------------------------------------------------------------------------------------------- inputs
def ztask_inputs(kind: int, B: int, n: int, seed: int, early: bool = True, power: bool = True, reach_id: int = None):
    """Inputs of one latent-task step (CPU float32 / int64), rows 0 .. BUILT - 1 the built edge envs when n >= BUILT."""
    g = torch.Generator().manual_seed(seed)
    body = torch.zeros(n, B, 13)
    body[..., 0:3] = torch.randn(n, B, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, B, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, B, 6, generator=g) * 2.0
    far = torch.rand(n, generator=g) < 0.3                      # coordinates 100 - 500 m
    body[far, :, 0:2] += (100.0 + 400.0 * torch.rand(int(far.sum()), 1, 2, generator=g))
    contact = torch.zeros(n, B, 3)
    hit = torch.rand(n, B, generator=g) < 0.05
    contact[hit] = torch.randn(int(hit.sum()), 3, generator=g) * 30.0
    term_h = 0.1 + 0.4 * torch.rand(B, generator=g)
    progress = torch.randint(0, MAX_LEN, (n,), generator=g)
    root = body[:, 0, 0:3]
    prev = root - torch.randn(n, 3, generator=g) * 0.1
    inp = dict(body=body, contact=contact, term_h=term_h, progress=progress, early=early, max_len=MAX_LEN, dt=DT, prev=prev,
               contact_mask=mask_of(SMPL_CONTACTS if B == 24 else SMPLX_CONTACTS), strike_mask=0)
    if kind == sf.SPEED:
        inp["tar_speed"] = 5.0 * torch.rand(n, generator=g)
        if power and B == 24:
            inp.update(dof_force=torch.randn(n, sf.NUM_DOF, generator=g) * 50.0, dof_vel=torch.randn(n, sf.NUM_DOF, generator=g) * 3.0,
                       power_c=0.0005)
    elif kind == sf.REACH:
        inp["tar_pos"] = root + torch.randn(n, 3, generator=g) * 0.5
        inp["reach_id"] = REACH_IDS[B][0] if reach_id is None else reach_id
    else:
        inp["strike_mask"] = mask_of(SMPL_STRIKE if B == 24 else SMPLX_STRIKE)
        tgt = torch.zeros(n, 13)
        tgt[:, 0:2] = root[:, 0:2] + torch.randn(n, 2, generator=g) * 3.0
        tgt[:, 2] = 0.9
        tgt[:, 3:7] = torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=-1)
        tgt[:, 7:13] = torch.randn(n, 6, generator=g)
        inp["target"] = tgt
        inp["tar_contact"] = torch.randn(n, 3, generator=g) * 40.0
    if n >= BUILT:
        _build_edges(kind, B, inp)
    return inp


def _build_edges(kind: int, B: int, inp):
    body, contact, prog = inp["body"], inp["contact"], inp["progress"]
    contact[:BUILT] = 0.0
    body[:BUILT, :, 2] = 0.9                                   # nobody below its termination height ...
    prog[:BUILT] = 10
    body[0, 0, 3:7] = torch.tensor([0.5, 0.5, -0.5, 0.5])       # the root's x axis exactly vertical: heading 0
    a = math.pi / 2 - 1e-3                                      # ... and within 1e-3 of vertical
    body[1, 0, 3:7] = torch.tensor([0.0, math.sin(a / 2), 0.0, math.cos(a / 2)])
    body[2, 0, 3:7] = -body[2, 0, 3:7].abs()                    # w < 0
    for r, p in zip(range(3, 10), (0, 1, 2, 3, 4, MAX_LEN - 2, MAX_LEN - 1)):
        prog[r] = p
        body[r, 5, 2] = 0.0                                     # fallen: a non-contact body low and pressing
        contact[r, 6, 0] = -0.2
    # force components exactly 0.1 (no contact) and 50 (no hard contact), negative included
    body[10, 5, 2] = 0.0
    contact[10, 6] = torch.tensor([0.1, -0.1, 0.1])
    if B == 52:
        body[11, 33, 2] = 0.0                                   # only a second-slot body is low ...
        contact[11, 45, 2] = 0.5                                # ... and only a second-slot body presses: fallen
        body[12, 40, 2] = 0.0                                   # a contact body of the second slot on the ground: not fallen
        contact[12, 40, 2] = 5.0
        contact[12, 47, 2] = 5.0
        body[12, 2, 2] = 0.0
        contact[13, 47, 0] = 0.5                                # height from the first slot, contact from the second
        body[13, 1, 2] = 0.0
    else:
        body[11, 5, 2] = 0.0
        contact[11, 6, 2] = 5.0
    root = body[:, 0, 0:3]
    inp["prev"][14] = root[14]                                  # prev_root_pos == root
    if kind == sf.STRIKE:
        tg, tc = inp["target"], inp["tar_contact"]
        tc[:BUILT] = 0.0
        tg[13, 0:2] = root[13, 0:2]                             # the target straight above the root
        tg[13:15, 3:7] = torch.tensor([0.0, 0.0, 0.0, 1.0])     # upright (rot_err 1): the velocity term decides the reward
        tg[15, 3:7] = torch.tensor(ROT_EDGE)
        tc[14] = torch.tensor([50.0, -50.0, 90.0])              # 50 N: not pushed
        hard = 35 if B == 52 else 20
        contact[14, hard, 1] = 70.0
        tc[15] = torch.tensor([-60.0, 0.0, 0.0])                # pushed while a strike body (allowed) presses
        sb = 45 if B == 52 else 20
        contact[15, sb if B == 52 else 21, 0] = -70.0
        if B == 52:
            contact[15, 33, 0] = 50.0                           # exactly 50 N on a non-strike body: not hard


def built_mask(n: int) -> torch.Tensor:
    m = torch.zeros(n, dtype=torch.bool)
    m[:min(n, BUILT)] = True
    return m


# ---------------------------------------------------------------------------------------------------------------- fp32 simulations
def heading_half32(q):
    """heading_half with its atan2(0, 0) branch: the inverse heading (0, 0, -hs, hc)."""
    x, y, z, w = q.unbind(-1)
    s = 2.0 * w * w - 1.0
    rx, ry = s + 2.0 * x * x, 2.0 * w * z + 2.0 * x * y
    n2 = rx * rx + ry * ry
    zero = ~(n2 > 0)
    inv = torch.rsqrt(torch.where(zero, torch.ones_like(n2), n2))
    ch, sh = rx * inv, ry * inv
    pos = ch >= 0
    c1 = torch.sqrt(0.5 * (1.0 + ch))
    s2 = torch.copysign(torch.sqrt(0.5 * (1.0 - ch)), sh)
    hc = torch.where(pos, c1, 0.5 * sh / s2)
    hs = torch.where(pos, 0.5 * sh / c1, s2)
    hs, hc = torch.where(zero, torch.zeros_like(hs), hs), torch.where(zero, torch.ones_like(hc), hc)
    return torch.stack([torch.zeros_like(hs), torch.zeros_like(hs), -hs, hc], -1)


def base_removed32(q, upright):
    return q if upright else qmul8_32(q, torch.tensor([-0.5, -0.5, -0.5, 0.5]).expand_as(q))


def self_obs32(body, upright, zshift=None):
    n, B = body.shape[0], body.shape[1]
    p, q, v, w = body[..., 0:3].clone(), body[..., 3:7], body[..., 7:10], body[..., 10:13]
    if zshift is not None:
        p[..., 2] = p[..., 2] - zshift[:, None]
    h = heading_half32(base_removed32(q[:, 0], upright))
    hb = h[:, None].expand(n, B, 4)
    pos = qrot32(hb[:, 1:], p[:, 1:] - p[:, :1])
    return torch.cat([p[:, 0, 2:3], pos.reshape(n, -1), six32(qmul8_32(hb, q)).reshape(n, -1), qrot32(hb, v).reshape(n, -1),
                      qrot32(hb, w).reshape(n, -1)], 1)


def sim_ztask(kind: int, B: int, inp, mut=None):
    """ztask_env<L> in float32: {"obs", "rew", "raw", "reset", "terminate"}."""
    body = inp["body"].float()[:, :B]
    n = body.shape[0]
    root, rq = body[:, 0, 0:3], body[:, 0, 3:7]
    obs = [self_obs32(body, B == 24 or mut == "self_raw_heading")]
    h = heading_half32(rq)
    prog = inp["progress"]
    raw = None
    if kind == sf.SPEED:
        d = qrot32(h, torch.tensor([1.0, 0.0, 0.0]).expand(n, 3))
        obs.append(torch.cat([d[:, :2], inp["tar_speed"][:, None]], 1))
        prev = inp["prev"][:, [1, 0]] if mut == "prev_swap" else inp["prev"][:, :2]
        v = (root[:, :2] - prev) / torch.tensor(inp["dt"])
        err = inp["tar_speed"] - v[:, 0]
        rew = torch.exp(-0.25 * (err * err + 0.1 * v[:, 1] * v[:, 1]))
        raw = rew[:, None].clone()
        if inp.get("dof_force") is not None:
            pw = -torch.tensor(np.float32(inp["power_c"])) * (inp["dof_force"] * inp["dof_vel"]).abs().sum(-1)
            if mut != "power_no_progress_zero":
                pw = torch.where(prog <= 3, torch.zeros_like(pw), pw)
            raw = torch.stack([rew, pw], 1)
            rew = rew + pw
    elif kind == sf.REACH:
        obs.append(qrot32(h, inp["tar_pos"] - root))
        rid = inp["reach_id"] & 31 if mut == "reach_slot0" else inp["reach_id"]
        d = inp["tar_pos"] - body[:, rid, 0:3]
        rew = torch.exp(-4.0 * (d * d).sum(-1))
    else:
        tg = inp["target"].float()
        tp, tq = tg[:, 0:3], tg[:, 3:7]
        rel = torch.stack([tp[:, 0] - root[:, 0], tp[:, 1] - root[:, 1], tp[:, 2]], 1)
        obs.append(torch.cat([qrot32(h, rel), six32(qmul8_32(h, tq)), qrot32(h, tg[:, 7:10]), qrot32(h, tg[:, 10:13])], 1))
        rot_err = 2.0 * tq[:, 3] * tq[:, 3] - 1.0 + 2.0 * tq[:, 2] * tq[:, 2]
        rot_r = torch.clamp(1.0 - rot_err, min=0.0)
        dxy = tp[:, 0:2] - root[:, 0:2]
        dn = torch.clamp(torch.sqrt((dxy * dxy).sum(-1)), min=1e-12)
        u = dxy / dn[:, None]
        v = (root[:, :2] - inp["prev"][:, :2]) / torch.tensor(inp["dt"])
        ds = u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]
        verr = torch.clamp(1.0 - ds, min=0.0)
        vel_r = torch.exp(-4.0 * verr * verr)
        vel_r = torch.where(ds < 0 if mut == "dir_speed_lt" else ds <= 0, torch.zeros_like(vel_r), vel_r)
        rew = 0.6 * rot_r + 0.4 * vel_r
        rew = torch.where(rot_err <= 0.2 if mut == "rot_err_le" else rot_err < 0.2, torch.ones_like(rew), rew)
    # reset
    cm = inp["contact_mask"] & 0xFFFFFFFF if mut == "mask32" else inp["contact_mask"]
    lim = 32 if mut == "fall_first_slot" else B
    bits = torch.tensor([bool((cm >> j) & 1) or j >= lim for j in range(B)])
    contact = ((inp["contact"][:, :B].abs() > 0.1).any(-1) & ~bits).any(-1)
    height = ((body[..., 2] < inp["term_h"][None, :B]) & ~bits).any(-1)
    failed = contact & height
    if kind == sf.STRIKE:
        sbits = torch.tensor([bool(((inp["contact_mask"] | inp["strike_mask"]) >> j) & 1) for j in range(B)])
        hard = ((inp["contact"][:, :B].abs() > 50.0).any(-1) & ~sbits).any(-1)
        tc = inp["tar_contact"].abs()
        failed = failed | (((tc[:, 0] > 50.0) | (tc[:, 1] > 50.0)) & hard)
    if not inp["early"]:
        failed = torch.zeros_like(failed)
    term = (failed & (prog > 1)).long()
    reset = torch.where(prog >= inp["max_len"] - 1, torch.ones_like(term), term)
    return {"obs": torch.cat(obs, 1), "rew": rew, "raw": raw, "reset": reset, "terminate": term,
            "power": inp.get("dof_force") is not None}


CASES = [("smpl reach", sf.REACH, 24), ("smpl speed", sf.SPEED, 24), ("smpl strike", sf.STRIKE, 24), ("smplx speed", sf.SPEED, 52),
         ("smplx reach", sf.REACH, 52), ("smplx strike", sf.STRIKE, 52)]


@pytest.mark.parametrize("early", [True, False])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_simulations_pass_every_link(case, early):
    tag, kind, B = case
    rep = sf.Report(tag)
    for rid in (REACH_IDS[B] if kind == sf.REACH else (None,)):
        inp = ztask_inputs(kind, B, 257, seed=3, early=early, reach_id=rid)
        ref = sf.ztask_ref(kind, B, inp)
        sf.check_step(rep, tag, kind, B, sim_ztask(kind, B, inp), ref, built=built_mask(257))
        if early:
            assert int(ref["terminate"][3:12].sum()) > 0 and int(ref["terminate"][:3].sum()) == 0
    assert all(r[1] < 1.0 for r in rep.rows)


MUTATIONS = [
    ("smplx speed", sf.SPEED, 52, "fall_first_slot", "terminate"),
    ("smplx strike", sf.STRIKE, 52, "fall_first_slot", "terminate"),
    ("smplx reach", sf.REACH, 52, "mask32", "terminate"),
    ("smplx speed", sf.SPEED, 52, "mask32", "terminate"),
    ("smplx reach", sf.REACH, 52, "reach_slot0", "reward"),
    ("smplx speed", sf.SPEED, 52, "self_raw_heading", "self body pos"),
    ("smpl strike", sf.STRIKE, 24, "rot_err_le", "reward"),
    ("smplx strike", sf.STRIKE, 52, "rot_err_le", "reward"),
    ("smpl strike", sf.STRIKE, 24, "dir_speed_lt", "reward"),
    ("smplx strike", sf.STRIKE, 52, "dir_speed_lt", "reward"),
    ("smpl speed", sf.SPEED, 24, "power_no_progress_zero", "reward raw power"),
    ("smpl speed", sf.SPEED, 24, "prev_swap", "reward raw speed"),
    ("smplx speed", sf.SPEED, 52, "prev_swap", "reward raw speed"),
]


@pytest.mark.parametrize("tag,kind,B,mut,link", MUTATIONS, ids=[f"{m[0]}-{m[3]}" for m in MUTATIONS])
def test_mutations_fail_their_link(tag, kind, B, mut, link):
    for rid in (REACH_IDS[B] if kind == sf.REACH else (None,)):
        inp = ztask_inputs(kind, B, 257, seed=3, reach_id=rid)
        ref = sf.ztask_ref(kind, B, inp)
        got = sim_ztask(kind, B, inp, mut=mut)
        if kind == sf.REACH and mut == "reach_slot0" and rid < 32:
            sf.check_step(None, tag, kind, B, got, ref, built=built_mask(257))      # the slot does not matter below 32
            continue
        with pytest.raises(sf.BoundError, match=f"^{tag} {link}"):
            sf.check_step(None, tag, kind, B, got, ref, built=built_mask(257))


def test_vertical_heading_is_exact():
    """rx = ry = 0 exactly: heading 0, decided (not ill-conditioned); the near-vertical root is well-conditioned too."""
    inp = ztask_inputs(sf.SPEED, 24, 32, seed=1)
    ref = sf.ztask_ref(sf.SPEED, 24, inp)
    assert not bool(ref["self"]["ill"][:3].any()) and not bool(ref["task ill"][:3].any())
    d, t = ref["task"]["speed dir"]
    assert d[0].tolist() == [1.0, 0.0] and float(t[0].max()) < 2e-6


def test_strike_edges_are_decided():
    for B in (24, 52):
        inp = ztask_inputs(sf.STRIKE, B, 64, seed=2)
        ref = sf.ztask_ref(sf.STRIKE, B, inp)
        assert bool(ref["rot_decided"][:BUILT].all()) and bool(ref["dir_decided"][[13, 14]].all())
        assert float(sf.rot_err_orders(inp["target"][15:16, 3:7]).max()) == sf.ROT_THRESH


# ---------------------------------------------------------------------------------------------------------------- small entry points
def test_reach_update_task_links():
    g = torch.Generator().manual_seed(4)
    n = 300
    prog, change = torch.randint(0, 50, (n,), generator=g), torch.randint(0, 50, (n,), generator=g)
    tar, rand, steps = torch.randn(n, 3, generator=g), torch.rand(n, 3, generator=g), torch.randint(10, 20, (n,), generator=g)
    ref = sf.reach_update_ref(prog, change, tar, rand, steps, 1.5, 0.4, 1.6)
    due = prog >= change
    got = torch.where(due[:, None], torch.stack([np.float32(1.5) * (2.0 * rand[:, 0] - 1.0), np.float32(1.5) * (2.0 * rand[:, 1] - 1.0),
                                                 (torch.tensor(np.float32(1.6)) - np.float32(0.4)) * rand[:, 2] + np.float32(0.4)], 1), tar)
    sf.check(None, "reach update target", got, *ref["target"])
    with pytest.raises(sf.BoundError, match="reach update target"):
        sf.check(None, "reach update target", torch.where(due[:, None], got, got + 1e-3), *ref["target"])


# ---------------------------------------------------------------------------------------------------------------- terrain
HS, VS = 0.1, 0.005


def terrain_inputs(n: int, seed: int, plane: bool = False, K: int = 10, P: int = 45, **opts):
    g = torch.Generator().manual_seed(seed)
    R, Cc = 160, 140
    hf = None if plane else torch.randint(-400, 400, (R, Cc), generator=g).to(torch.int16)
    body = torch.zeros(n, 24, 13)
    center = torch.stack([torch.rand(n, generator=g) * R * HS, torch.rand(n, generator=g) * Cc * HS], 1)
    body[..., 0:2] = center[:, None] + torch.randn(n, 24, 2, generator=g) * 0.3
    body[..., 2] = 0.9 + torch.randn(n, 24, generator=g) * 0.2
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 24, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 24, 6, generator=g)
    root = body[:, 0].clone()
    root[:, 0:3] += torch.randn(n, 3, generator=g) * 0.5          # the actor root is not the rigid-body root
    root[:, 3:7] = torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=-1)
    verts = torch.zeros(n, sf.TRAJ_VERTS, 3)
    steps = torch.randn(n, sf.TRAJ_VERTS - 1, 2, generator=g) * 0.3
    verts[:, 0, :2] = body[:, 0, :2] + torch.randn(n, 2, generator=g) * 2.0
    verts[:, 1:, :2] = verts[:, :1, :2] + torch.cumsum(steps, 1)
    contact = torch.zeros(n, 24, 3)
    hit = torch.rand(n, 24, generator=g) < 0.1
    contact[hit] = torch.randn(int(hit.sum()), 3, generator=g) * 40.0
    pts = torch.zeros(P, 3)
    pts[:, 0:2] = (torch.rand(P, 2, generator=g) - 0.5) * 2.0       # the square sensor's 2 m extent
    cpts = torch.tensor([[x, y, 0.0] for x in (-0.1, 0.0, 0.1) for y in (-0.2, 0.0, 0.2)])
    inp = dict(body=body, root=root, progress=torch.randint(0, 320, (n,), generator=g), contact=contact, contact_mask=mask_of(SMPL_CONTACTS),
               early=True, no_collision=False, fuzzy=False, power_reward=True, upright=True, use_center_height=True, num_traj_samples=K,
               height_points=pts, center_points=cpts, head_id=13, dt=DT, traj_dt=0.1, sample_dt=0.5, fail_dist=4.0, power_c=0.0005,
               verts=verts, hf=hf, hscale=HS, vscale=VS, dof_force=torch.randn(n, sf.NUM_DOF, generator=g) * 50.0,
               dof_vel=torch.randn(n, sf.NUM_DOF, generator=g) * 3.0, max_len=300)
    inp.update(opts)
    if n >= BUILT:
        _terrain_edges(inp, R, Cc)
    return inp


def _terrain_edges(inp, R, Cc):
    body, root, verts, contact, prog = inp["body"], inp["root"], inp["verts"], inp["contact"], inp["progress"]
    contact[:BUILT] = 0.0
    # the rigid-body root on the trajectory's start (not far), progress 0 (t = 0) and past the end
    for r in range(BUILT):
        verts[r, :, :2] = body[r, 0, :2] + torch.tensor([0.01 * r, 0.0])
        verts[r, 1:, :2] += torch.cumsum(torch.full((sf.TRAJ_VERTS - 1, 2), 1e-3), 0)
    prog[0], prog[1] = 0, 100000
    # heads past all four map edges and in (-h, 0)
    head = inp["head_id"]
    body[2, head, 0:2] = torch.tensor([-5.0, 3.0])
    body[3, head, 0:2] = torch.tensor([R * HS + 5.0, 3.0])
    body[4, head, 0:2] = torch.tensor([3.0, -5.0])
    body[5, head, 0:2] = torch.tensor([3.0, Cc * HS + 5.0])
    body[6, head, 0:2] = torch.tensor([-0.05, -0.05])
    # height differences beyond +-3 m
    root[7, 2] = 40.0
    root[8, 2] = -40.0
    # the force sum exactly 50 (not fallen) and just over it (fallen), at progress 2
    prog[9] = prog[10] = 2
    contact[9, 5] = torch.tensor([30.0, 0.0, 0.0])
    contact[9, 6] = torch.tensor([0.0, -40.0, 0.0])
    contact[10, 5] = torch.tensor([-51.0, 0.0, 0.0])
    contact[11, 7] = torch.tensor([1000.0, 0.0, 0.0])            # a contact body: not summed
    # far from the rigid-body root, while the actor root is on the trajectory; and the reverse
    body[12, 0, 0:2] = verts[12, 0, :2] + 10.0
    root[12, 0:2] = verts[12, 0, :2]
    root[13, 0:2] = verts[13, 0, :2] + 10.0
    prog[12] = prog[13] = 0
    root[14, 3:7] = -root[14, 3:7].abs()                          # w < 0


def sim_traj32(verts, t, traj_dur):
    phase = torch.clamp(t / traj_dur, 0.0, 1.0)
    seg = phase * float(sf.TRAJ_VERTS - 1)
    i0, i1 = torch.floor(seg).long(), torch.ceil(seg).long()
    b = (seg - i0.float())[..., None]
    g = lambda i: torch.gather(verts, 1, i.reshape(verts.shape[0], -1, 1).expand(-1, -1, 3))
    return (1.0 - b) * g(i0) + b * g(i1)


def heading_quat_ref32(q, inverse):
    x, y, z, w = q.unbind(-1)
    s = 2.0 * (w * w) - 1.0
    rx, ry = s + (x * x) * 2.0, (z * w) * 2.0 + (y * x) * 2.0
    h = torch.atan2(ry, rx)
    if inverse:
        h = -h
    sn, cs = torch.sin(h * 0.5), torch.cos(h * 0.5)
    nn = torch.clamp(torch.sqrt(sn * sn + cs * cs), min=1e-9)
    return torch.stack([torch.zeros_like(sn), torch.zeros_like(sn), sn / nn, cs / nn], -1)


def quat_apply32(q, b):
    u = q[..., :3]
    t = torch.cross(u, b, dim=-1) * 2.0
    return b + q[..., 3:] * t + torch.cross(u, t, dim=-1)


def sample_height32(hf, x, y, mut=None):
    if hf is None:
        return torch.zeros_like(x)
    R, Cc = hf.shape
    px = (x / np.float32(HS)).trunc().long().clamp(0, R - 2)
    py = (y / np.float32(HS)).trunc().long().clamp(0, Cc - 2)
    h1, h2 = hf.long()[px, py], hf.long()[px + 1, py + 1]
    return (torch.maximum(h1, h2) if mut == "max_cell" else torch.minimum(h1, h2)).float() * np.float32(VS)


def height_at32(hf, q, pts, origin, mut=None):
    r = quat_apply32(q[:, None].expand(-1, pts.shape[0], 4), pts[None].expand(q.shape[0], -1, 3))
    return sample_height32(hf, r[..., 0] + origin[:, None, 0], r[..., 1] + origin[:, None, 1], mut)


def center32(hf, pts, q, pos, upright):
    qb = base_removed32(q, upright)
    nn = torch.clamp(torch.sqrt(qb[:, 2] * qb[:, 2] + qb[:, 3] * qb[:, 3]), min=1e-9)
    qy = torch.stack([torch.zeros_like(nn), torch.zeros_like(nn), qb[:, 2] / nn, qb[:, 3] / nn], -1)
    return height_at32(hf, qy, pts, pos).sum(-1) / pts.shape[0]


def sim_terrain(inp, flags=7, mut=None):
    body, root = inp["body"], inp["root"]
    n = body.shape[0]
    upright = inp["upright"]
    prog = inp["progress"]
    t_now = prog.float() * torch.tensor(inp["dt"], dtype=torch.float32)
    dur = torch.tensor(np.float32((sf.TRAJ_VERTS - 1 if mut == "phase_segs" else sf.TRAJ_VERTS) * inp["traj_dt"]))
    tar = sim_traj32(inp["verts"], t_now[:, None], dur)[:, 0]
    out = {"power_reward": inp["power_reward"]}
    if flags & 1:
        d = tar[:, :2] - root[:, :2]
        err = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
        if inp["fuzzy"]:
            err = torch.where(err < 0.0025, torch.zeros_like(err), err)
        loc = torch.exp(-2.0 * err)
        power = -torch.tensor(np.float32(inp["power_c"])) * (inp["dof_force"] * inp["dof_vel"]).abs().sum(-1)
        out["rew"] = loc + power if inp["power_reward"] else loc
        out["raw"] = torch.stack([loc, power], 1)
    if flags & 2:
        cm = inp["contact_mask"]
        bits = torch.tensor([bool((cm >> j) & 1) for j in range(24)])
        sel = bits if mut == "force_contact_bodies" else ~bits
        f = inp["contact"] * sel[None, :, None]
        s = torch.zeros(n, 3)
        for j in range(24):
            s = s + f[:, j]
        nrm = torch.sqrt(s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1] + s[:, 2] * s[:, 2])
        fallen = (nrm > 50.0) & (prog > 1)
        src = root if mut == "far_actor_root" else body[:, 0]
        d = tar[:, :2] - src[:, :2]
        far = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] > torch.tensor(np.float32(inp["fail_dist"])) ** 2
        term = ((fallen | far) & (inp["early"] and not inp["no_collision"])).long()
        out["terminate"] = term
        out["reset"] = torch.where(prog >= inp["max_len"] - 1, torch.ones_like(term), term)
    if flags & 4:
        hf = inp["hf"]
        src = root if mut == "center_actor_root" else body[:, 0]
        c_self = center32(hf, inp["center_points"], src[:, 3:7], src[:, 0:3], upright)
        obs = [self_obs32(body, upright, zshift=c_self)]
        K = inp["num_traj_samples"]
        tk = t_now[:, None] + torch.arange(K, dtype=torch.float32)[None] * torch.tensor(np.float32(inp["sample_dt"]))
        tp = sim_traj32(inp["verts"], tk, dur)
        hq = heading_quat_ref32(base_removed32(root[:, 3:7], upright), True)
        lt = qrot32(hq[:, None].expand(n, K, 4), tp - root[:, None, 0:3])
        obs.append(lt[..., :2].reshape(n, -1))
        ref_h = center32(hf, inp["center_points"], root[:, 3:7], root[:, 0:3], upright) if inp["use_center_height"] else root[:, 2]
        head = body[:, inp["head_id"]]
        hq = heading_quat_ref32(base_removed32(head[:, 3:7], upright), False)
        m = height_at32(hf, hq, inp["height_points"], head[:, 0:3], mut)
        dh = ref_h[:, None] - m
        obs.append((dh if mut == "unclipped" else torch.clamp(dh, -3.0, 3.0)) * 5.0)
        out["obs"] = torch.cat(obs, 1)
    return out


@pytest.mark.parametrize("variant", ["default", "plane", "fuzzy", "no_center", "not_upright", "no_collision", "no_power"])
def test_terrain_simulation_passes_every_link(variant):
    opts = {"fuzzy": dict(fuzzy=True), "no_center": dict(use_center_height=False), "not_upright": dict(upright=False),
            "no_collision": dict(no_collision=True), "no_power": dict(power_reward=False)}.get(variant, {})
    inp = terrain_inputs(257, seed=5, plane=variant == "plane", **opts)
    rep = sf.Report(f"terrain {variant}")
    ref = sf.terrain_ref(inp, 7)
    got = sim_terrain(inp)
    sf.check_terrain(rep, "terrain", 7, got, ref, inp["num_traj_samples"], built=built_mask(257))
    if variant == "default":
        assert got["terminate"][[10, 12]].tolist() == [1, 1] and got["terminate"][[9, 11, 13]].tolist() == [0, 0, 0]
        assert not bool((ref["term_lo"] != ref["term_hi"])[:BUILT].any())


TERRAIN_MUTATIONS = [("max_cell", "heights"), ("center_actor_root", "self root h"), ("phase_segs", "reward"), ("unclipped", "heights"),
                     ("force_contact_bodies", "terminate"), ("far_actor_root", "terminate")]


@pytest.mark.parametrize("mut,link", TERRAIN_MUTATIONS, ids=[m[0] for m in TERRAIN_MUTATIONS])
def test_terrain_mutations_fail_their_link(mut, link):
    inp = terrain_inputs(257, seed=5)
    ref = sf.terrain_ref(inp, 7)
    with pytest.raises(sf.BoundError, match=f"^terrain {link}"):
        sf.check_terrain(None, "terrain", 7, sim_terrain(inp, mut=mut), ref, inp["num_traj_samples"], built=built_mask(257))
