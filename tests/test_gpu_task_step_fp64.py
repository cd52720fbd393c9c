"""The task step kernels element-wise against their float64 references (tests/step_fp64.py), through every entry point: the step, the
list observation and the rollout step of reach (SMPL), speed with and without the power term and strike (SMPL), SMPL-X speed and
SMPL-X reach / strike; the pedestrian terrain step under every flag subset, with an env list, and its rollout step; the reach task
update and the imitation AMP row.  Inputs come as Isaac Gym lays them out (extra bodies per env, the target's contact appended to the
contact tensor, interleaved dof state, observation rows wider than the layout), with the built edge envs of
tests/test_task_step_fp64_cpu.py in the first rows.  With -s every link's largest err / tol and ambiguous share is printed."""
import ctypes as C

import pytest
import torch

from tests import reset_fp64 as rf
from tests import step_fp64 as sf
from tests.test_task_step_fp64_cpu import BUILT, CASES, REACH_IDS, built_mask, terrain_inputs, ztask_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [1, 257, 2051, 16384]
EXTRA = {24: 26 - 24, 52: 53 - 52}       # bodies per env beyond the humanoid's (SMPL strike: 26, SMPL-X: 53)
PAD = 5                                  # observation rows wider than the layout
SENTINEL = -7.0


def _lib():
    from pulse_b200 import _lib as L
    return L, L.load()


def _stream():
    from pulse_b200 import _lib as L
    return L.current_stream(DEV)


class Views:
    """Device views of one latent-task batch as Isaac Gym shapes them."""

    def __init__(self, kind, B, inp, width):
        n = inp["body"].shape[0]
        self.n = n
        self.rb = torch.full((n, B + EXTRA[B], 13), 5.0, device=DEV)
        self.rb[:, :B] = inp["body"].to(DEV)
        self.cf = torch.zeros(n, B + 1, 3, device=DEV)
        self.cf[:, :B] = inp["contact"].to(DEV)
        self.term_h = inp["term_h"].to(DEV)
        self.prog = inp["progress"].to(DEV)
        self.prev = inp["prev"].to(DEV)
        self.obs = torch.full((n, width + PAD), SENTINEL, device=DEV)
        self.rew = torch.full((n,), SENTINEL, device=DEV)
        self.raw = torch.full((n, 3), SENTINEL, device=DEV)
        self.reset = torch.full((n,), -3, dtype=torch.int64, device=DEV)
        self.term = torch.full((n,), -3, dtype=torch.int64, device=DEV)
        self.tar_speed = inp["tar_speed"].to(DEV) if "tar_speed" in inp else None
        self.tar_pos = inp["tar_pos"].to(DEV) if "tar_pos" in inp else None
        if kind == sf.STRIKE:
            roots = torch.zeros(n, 2, 13, device=DEV)
            roots[:, 1] = inp["target"].to(DEV)
            self.ts = roots[:, 1]
            self.cf[:, B] = inp["tar_contact"].to(DEV)
            self.tcf = self.cf[:, B]
        if inp.get("dof_force") is not None:
            ds = torch.zeros(n, sf.NUM_DOF, 2, device=DEV)
            ds[..., 1] = inp["dof_vel"].to(DEV)
            self.dof_state = ds
            self.dof_force = inp["dof_force"].to(DEV)


def _args(kind, B, inp, v: Views, power: bool):
    L, _ = _lib()
    common = dict(enable_early_termination=int(inp["early"]), body_state=v.rb.data_ptr(), body_env_stride=v.rb.stride(0),
                  contact_forces=v.cf.data_ptr(), contact_env_stride=v.cf.stride(0), termination_heights=v.term_h.data_ptr(),
                  contact_body_mask=inp["contact_mask"], progress_buf=v.prog.data_ptr(), max_episode_length=inp["max_len"],
                  obs_buf=v.obs.data_ptr(), obs_stride=v.obs.stride(0), rew_buf=v.rew.data_ptr(), reset_buf=v.reset.data_ptr(),
                  terminate_buf=v.term.data_ptr())
    if B == 24 and kind == sf.REACH:
        return "reach", L.ReachStepArgs(tar_pos=v.tar_pos.data_ptr(), reach_body_id=inp["reach_id"], **common)
    if B == 24:
        a = L.ZTaskStepArgs(kind=kind, strike_body_mask=inp["strike_mask"], prev_root_pos=v.prev.data_ptr(), dt=inp["dt"], **common)
        if kind == sf.SPEED:
            a.tar_speed, a.reward_raw, a.raw_stride = v.tar_speed.data_ptr(), v.raw.data_ptr(), v.raw.stride(0)
            if power:
                a.dof_force, a.dof_force_stride, a.power_coefficient = v.dof_force.data_ptr(), v.dof_force.stride(0), inp["power_c"]
                dv = v.dof_state[..., 1]
                a.dof_vel, a.dof_env_stride, a.dof_elem_stride = dv.data_ptr(), dv.stride(0), dv.stride(1)
        else:
            a.target_states, a.target_env_stride = v.ts.data_ptr(), v.ts.stride(0)
            a.tar_contact_forces, a.tar_contact_env_stride = v.tcf.data_ptr(), v.tcf.stride(0)
        return "ztask", a
    if kind == sf.SPEED:
        return "smplx_speed", L.SmplxSpeedStepArgs(prev_root_pos=v.prev.data_ptr(), dt=inp["dt"], tar_speed=v.tar_speed.data_ptr(),
                                                   reward_raw=v.raw.data_ptr(), raw_stride=v.raw.stride(0), **common)
    a = L.SmplxTargetStepArgs(kind=kind, strike_body_mask=inp["strike_mask"], **common)
    if kind == sf.REACH:
        a.reach_body_id, a.tar_pos = inp["reach_id"], v.tar_pos.data_ptr()
    else:
        a.prev_root_pos, a.dt = v.prev.data_ptr(), inp["dt"]
        a.target_states, a.target_env_stride = v.ts.data_ptr(), v.ts.stride(0)
        a.tar_contact_forces, a.tar_contact_env_stride = v.tcf.data_ptr(), v.tcf.stride(0)
    return "smplx_target", a


def _got(v: Views, kind, B, power):
    return {"obs": v.obs.cpu(), "rew": v.rew.cpu(), "reset": v.reset.cpu(), "terminate": v.term.cpu(),
            "raw": v.raw.cpu()[:, :2 if power else 1] if kind == sf.SPEED else None, "power": power}


def _width(kind, B):
    return sf.self_obs_width(B) + (3 if kind != sf.STRIKE else 15)


def _run_case(rep, tag, kind, B, n, seed, early=True, power=True, reach_id=None):
    L, lib = _lib()
    inp = ztask_inputs(kind, B, n, seed, early=early, power=power, reach_id=reach_id)
    power = power and inp.get("dof_force") is not None
    if not power:
        inp.pop("dof_force", None)
    ref = sf.ztask_ref(kind, B, inp)
    built = built_mask(n)
    width = _width(kind, B)
    # the step
    v = Views(kind, B, inp, width)
    name, a = _args(kind, B, inp, v, power)
    L.check(getattr(lib, f"pulse_{name}_step")(C.byref(a), n, _stream()), name)
    torch.cuda.synchronize()
    got = _got(v, kind, B, power)
    sf.check_step(rep, tag, kind, B, got, ref, built)
    assert bool((got["obs"][:, width:] == SENTINEL).all()), f"{tag}: columns past the row written"
    if kind == sf.SPEED:
        assert bool((v.raw.cpu()[:, 2] == SENTINEL).all()), f"{tag}: reward_raw written past its columns"
        if not power and B == 24:
            assert bool((v.raw.cpu()[:, 1] == SENTINEL).all()), f"{tag}: power column written without the power term"
    # the list observation: the listed rows as the step wrote them, nothing else
    lst = torch.arange(0, n, 3, device=DEV)
    count = torch.tensor([lst.numel()], dtype=torch.int32, device=DEV)
    step_obs = v.obs.clone()
    v.obs.fill_(SENTINEL)
    before = {k: getattr(v, k).clone() for k in ("rew", "reset", "term")}
    L.check(getattr(lib, f"pulse_{name}_obs_list")(C.byref(a), lst.data_ptr(), count.data_ptr(), n, _stream()), name)
    torch.cuda.synchronize()
    keep = torch.ones(n, dtype=torch.bool, device=DEV)
    keep[lst] = False
    if B == sf.SMPL:
        assert torch.equal(v.obs[lst], step_obs[lst]), f"{tag}: list rows differ from the step's"
    else:   # the SMPL-X instantiations agree with the step to the last bit of a few self-observation columns only
        li = lst.cpu()
        sf.check_obs(rep, f"{tag} list", kind, B, v.obs.cpu()[li], {**ref, "self": {k: (x[0][li], x[1][li]) if k != "ill" else x[li]
                                                                                    for k, x in ref["self"].items()},
                                                                 "task": {k: (x[0][li], x[1][li]) for k, x in ref["task"].items()},
                                                                 "task ill": ref["task ill"][li]}, built[li])
    assert bool((v.obs[keep] == SENTINEL).all()), f"{tag}: the list observation wrote an unlisted row"
    for k, t in before.items():
        assert torch.equal(getattr(v, k), t), f"{tag}: the list observation wrote {k}"
    # the rollout step: progress += 1 first, the step's rows, dones = float(reset)
    v2 = Views(kind, B, inp, width)
    v2.prog -= 1
    _, a2 = _args(kind, B, inp, v2, power)
    dones = torch.full((n,), SENTINEL, device=DEV)
    L.check(getattr(lib, f"pulse_{name}_rollout_step")(C.byref(a2), dones.data_ptr(), n, _stream()), name)
    torch.cuda.synchronize()
    assert torch.equal(v2.prog.cpu(), inp["progress"]), f"{tag}: rollout progress"
    g2 = _got(v2, kind, B, power)
    sf.check_step(rep, f"{tag} rollout", kind, B, g2, ref, built)
    for k in ("obs", "rew", "reset", "terminate") if B == sf.SMPL else ("reset", "terminate"):
        assert torch.equal(g2[k], got[k]), f"{tag}: rollout {k} differs from the step's"
    assert torch.equal(dones.cpu(), g2["reset"].float())
    return ref


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_latent_task_steps(case, n, capsys):
    tag, kind, B = case
    rep = sf.Report(f"{tag} n={n}")
    variants = [dict(reach_id=r) for r in REACH_IDS[B]] if kind == sf.REACH else [{}]
    if kind == sf.SPEED and B == 24:
        variants = [dict(power=True), dict(power=False)]
    variants = variants + [dict(variants[0], early=False)]
    for i, kw in enumerate(variants):
        ref = _run_case(rep, tag, kind, B, n, seed=n + 11 * i, **kw)
        if n >= BUILT and kw.get("early", True):
            # the built envs are decided exactly: falls where they were built, none elsewhere among them
            assert int(ref["terminate"][3:5].sum()) == 0 and int(ref["terminate"][5:8].sum()) == 3
            if kind == sf.STRIKE:
                rd, dd = ref["rot_decided"], ref["dir_decided"]
                assert bool(rd[:BUILT].all()) and bool(dd[[13, 14]].all())
    with capsys.disabled():
        print("\n" + rep.text())


# ---------------------------------------------------------------------------------------------------------------- small entry points
def test_reach_update_task():
    L, lib = _lib()
    g = torch.Generator().manual_seed(9)
    n = 2051
    prog, change = torch.randint(0, 50, (n,), generator=g), torch.randint(0, 50, (n,), generator=g)
    tar, rand, steps = torch.randn(n, 3, generator=g), torch.rand(n, 3, generator=g), torch.randint(10, 20, (n,), generator=g)
    prog[:3], change[:3] = torch.tensor([5, 5, 0]), torch.tensor([5, 6, 0])      # progress == change: due; one below: not
    rand[0] = torch.tensor([0.0, 1.0, 1.0])
    ref = sf.reach_update_ref(prog, change, tar, rand, steps, 1.5, 0.4, 1.6)
    d = {k: t.to(DEV).contiguous() for k, t in dict(prog=prog, change=change, tar=tar, rand=rand, steps=steps).items()}
    L.check(lib.pulse_reach_update_task(d["prog"].data_ptr(), d["change"].data_ptr(), d["tar"].data_ptr(), d["rand"].data_ptr(),
                                        d["steps"].data_ptr(), C.c_float(1.5), C.c_float(0.4), C.c_float(1.6), n, _stream()), "update")
    torch.cuda.synchronize()
    rep = sf.Report("reach update task")
    sf.check(rep, "reach update target", d["tar"].cpu(), *ref["target"])
    sf.check_exact(rep, "reach update kept targets", d["tar"].cpu()[~ref["due"]], tar[~ref["due"]])
    sf.check_exact(rep, "reach update change steps", d["change"].cpu(), ref["change"])
    assert bool(ref["due"][0]) and not bool(ref["due"][1])
    print("\n" + rep.text())


@pytest.mark.parametrize("n", [1, 2051])
def test_amp_obs(n):
    L, lib = _lib()
    g = torch.Generator().manual_seed(n)
    S = 10
    body = torch.zeros(n, 26, 13)
    body[..., 0:3] = torch.randn(n, 26, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 26, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 26, 6, generator=g)
    dof = torch.randn(n, 69, 2, generator=g)
    dof[:, :3, 0] = 0.0                                     # a joint at exactly zero rotation: the identity branch
    buf = torch.randn(n, S, 196, generator=g).to(DEV)
    old = buf.clone()
    rb, ds = body.to(DEV), dof.to(DEV)
    a = L.AmpObsArgs(body_state=rb.data_ptr(), body_env_stride=rb.stride(0), dof_pos=ds[..., 0].data_ptr(), dof_vel=ds[..., 1].data_ptr(),
                     dof_env_stride=ds.stride(0), dof_elem_stride=2, amp_obs_buf=buf.data_ptr(), num_steps=S, shift_history=1)
    L.check(lib.pulse_amp_obs(C.byref(a), n, _stream()), "amp")
    torch.cuda.synchronize()
    rep = sf.Report("amp obs")
    rf.check_amp(rep, "amp obs", buf[:, 0].cpu(), sf.amp_obs_ref(body, dof[..., 0], dof[..., 1]))
    sf.check_exact(rep, "amp obs history shift", buf[:, 1:].cpu(), old[:, :-1].cpu())
    print("\n" + rep.text())


# ---------------------------------------------------------------------------------------------------------------- terrain
class TerrainViews:
    def __init__(self, inp, width):
        n = inp["body"].shape[0]
        self.rb = torch.full((n, 26, 13), 5.0, device=DEV)
        self.rb[:, :24] = inp["body"].to(DEV)
        roots = torch.zeros(n, 2, 13, device=DEV)
        roots[:, 0] = inp["root"].to(DEV)
        self.root = roots[:, 0]
        self.cf = torch.zeros(n, 26, 3, device=DEV)
        self.cf[:, :24] = inp["contact"].to(DEV)
        self.prog = inp["progress"].to(DEV)
        self.verts = inp["verts"].to(DEV).contiguous()
        self.hf = inp["hf"].to(DEV).contiguous() if inp["hf"] is not None else None
        self.hp, self.cp = inp["height_points"].to(DEV).contiguous(), inp["center_points"].to(DEV).contiguous()
        ds = torch.zeros(n, sf.NUM_DOF, 2, device=DEV)
        ds[..., 1] = inp["dof_vel"].to(DEV)
        self.dv = ds[..., 1]
        self.df = inp["dof_force"].to(DEV)
        self.obs = torch.full((n, width + PAD), SENTINEL, device=DEV)
        self.rew = torch.full((n,), SENTINEL, device=DEV)
        self.raw = torch.full((n, 2), SENTINEL, device=DEV)
        self.reset = torch.full((n,), -3, dtype=torch.int64, device=DEV)
        self.term = torch.full((n,), -3, dtype=torch.int64, device=DEV)

    def args(self, inp, flags):
        L, _ = _lib()
        hf = self.hf
        return L.TerrainStepArgs(
            flags=flags, upright=int(inp["upright"]), body_state=self.rb.data_ptr(), body_env_stride=self.rb.stride(0),
            root_states=self.root.data_ptr(), root_env_stride=self.root.stride(0), progress_buf=self.prog.data_ptr(),
            max_episode_length=inp["max_len"], contact_forces=self.cf.data_ptr(), contact_env_stride=self.cf.stride(0),
            contact_body_mask=inp["contact_mask"], enable_early_termination=int(inp["early"]), no_collision_check=int(inp["no_collision"]),
            fuzzy_target=int(inp["fuzzy"]), power_reward=int(inp["power_reward"]), num_traj_samples=inp["num_traj_samples"],
            num_height_points=self.hp.shape[0], num_center_points=self.cp.shape[0], head_body_id=inp["head_id"],
            use_center_height=int(inp["use_center_height"]), dt=inp["dt"], traj_dur=sf.TRAJ_VERTS * inp["traj_dt"],
            traj_sample_timestep=inp["sample_dt"], fail_dist=inp["fail_dist"], power_coefficient=inp["power_c"],
            traj_verts=self.verts.data_ptr(), heightfield=hf.data_ptr() if hf is not None else None,
            hf_rows=hf.shape[0] if hf is not None else 0, hf_cols=hf.shape[1] if hf is not None else 0, horizontal_scale=inp["hscale"],
            vertical_scale=inp["vscale"], height_points=self.hp.data_ptr(), center_points=self.cp.data_ptr(), dof_force=self.df.data_ptr(),
            dof_force_stride=self.df.stride(0), dof_vel=self.dv.data_ptr(), dof_env_stride=self.dv.stride(0), dof_elem_stride=self.dv.stride(1),
            obs_buf=self.obs.data_ptr(), obs_stride=self.obs.stride(0), rew_buf=self.rew.data_ptr(), reward_raw=self.raw.data_ptr(),
            raw_stride=self.raw.stride(0), reset_buf=self.reset.data_ptr(), terminate_buf=self.term.data_ptr())

    def got(self, inp):
        return {"obs": self.obs.cpu(), "rew": self.rew.cpu(), "raw": self.raw.cpu(), "reset": self.reset.cpu(), "terminate": self.term.cpu(),
                "power_reward": inp["power_reward"]}


TERRAIN_VARIANTS = {
    "default": {}, "plane": dict(plane=True), "fuzzy": dict(fuzzy=True), "no_center_height": dict(use_center_height=False),
    "not_upright": dict(upright=False), "no_collision_check": dict(no_collision=True), "no_power_reward": dict(power_reward=False),
    "no_early_termination": dict(early=False), "one_sample_37_points": dict(K=1, P=37), "32_samples_70_points": dict(K=32, P=70),
}


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("variant", list(TERRAIN_VARIANTS))
def test_terrain_step(variant, n, capsys):
    L, lib = _lib()
    inp = terrain_inputs(n, seed=n + 3, **TERRAIN_VARIANTS[variant])
    K = inp["num_traj_samples"]
    width = 358 + 2 * K + inp["height_points"].shape[0]
    ref = sf.terrain_ref(inp, 7)
    built = built_mask(n)
    rep = sf.Report(f"terrain {variant} n={n}")
    full = TerrainViews(inp, width)
    a = full.args(inp, 7)
    L.check(lib.pulse_terrain_step(C.byref(a), n, _stream()), "terrain")
    torch.cuda.synchronize()
    got = full.got(inp)
    sf.check_terrain(rep, "terrain", 7, got, ref, K, built)
    assert bool((got["obs"][:, width:] == SENTINEL).all())
    if n >= BUILT and variant == "default":
        assert got["terminate"][[10, 12]].tolist() == [1, 1] and got["terminate"][[9, 11, 13]].tolist() == [0, 0, 0]
        assert not bool((ref["term_lo"] != ref["term_hi"])[:BUILT].any())
    # every flag subset writes its own outputs, bit-identical to the full step's, and nothing else
    outs = {1: ("rew", "raw"), 2: ("reset", "term"), 4: ("obs",)}
    for flags in range(1, 7):
        v = TerrainViews(inp, width)
        L.check(lib.pulse_terrain_step(C.byref(v.args(inp, flags)), n, _stream()), "terrain flags")
        torch.cuda.synchronize()
        for bit, names in outs.items():
            for k in names:
                want = getattr(full, k) if flags & bit else getattr(TerrainViews(inp, width), k)
                assert torch.equal(getattr(v, k), want), f"flags {flags}: {k}"
    # the observation over an env list with a device count: the listed rows, nothing else
    if n > 1:
        v = TerrainViews(inp, width)
        ids = torch.arange(n - 1, -1, -5, device=DEV)
        cnt = torch.tensor([ids.numel()], dtype=torch.int32, device=DEV)
        a = v.args(inp, 4)
        a.env_ids, a.env_count = ids.data_ptr(), cnt.data_ptr()
        L.check(lib.pulse_terrain_step(C.byref(a), n, _stream()), "terrain list")
        torch.cuda.synchronize()
        keep = torch.ones(n, dtype=torch.bool, device=DEV)
        keep[ids] = False
        assert torch.equal(v.obs[ids], full.obs[ids]) and bool((v.obs[keep] == SENTINEL).all())
    # the rollout step
    v = TerrainViews(inp, width)
    v.prog -= 1
    dones = torch.full((n,), SENTINEL, device=DEV)
    L.check(lib.pulse_terrain_rollout_step(C.byref(v.args(inp, 7)), dones.data_ptr(), n, _stream()), "terrain rollout")
    torch.cuda.synchronize()
    assert torch.equal(v.prog.cpu(), inp["progress"])
    g2 = v.got(inp)
    sf.check_terrain(rep, "terrain rollout", 7, g2, ref, K, built)
    for k in ("obs", "rew", "raw", "reset", "terminate"):
        assert torch.equal(g2[k], got[k]), f"rollout {k}"
    assert torch.equal(dones.cpu(), g2["reset"].float())
    with capsys.disabled():
        print("\n" + rep.text())
