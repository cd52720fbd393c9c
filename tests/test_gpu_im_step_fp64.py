"""The fused imitation step (pulse_im_step, pulse_im_track_step) and the general task observation (pulse_im_task_obs) element-wise
against the float64 references of tests/step_fp64.py, link by link, at the shapes and edges where the kernels can go wrong: env counts
below one group of 8, a ragged last group and the benchmark's 16384 (every CTA wraps its plan ring and stage ring), clips at 24 to
120 fps (rows needing four distinct frame records, the fourth read straight from global memory), obs rows in all four 16-byte phases,
body rows only 4-byte aligned, strided dof velocities, staged flags, device-side env counts, and built edge envs in the first rows.
Run with -s for the margin of every link."""
import ctypes as C

import pytest
import torch

from tests import step_fp64 as sf
from tests.test_im_step_fp64_cpu import (BUILT, DEFAULT_RESET_BODIES, MIXED_RATES, TASK_CASES, config, im_inputs, im_tables, mask_of,
                                         nonuniform_term, table_dict, task_obs_inputs)

pytestmark = pytest.mark.gpu
SENT = -9.0


def _dev():
    return torch.device("cuda:0")


def _mlib(tb):
    from pulse_b200.motion_lib import MotionLibB200
    return MotionLibB200.from_tables(table_dict(tb), device=_dev())


def run_step(ml, cfg, inp, *, bodies=24, obs_stride=None, interleaved=True, env_ids=None, env_count=None, track=None, raw_width=None):
    """One HumanoidImCompute.step on device copies of inp, every output buffer filled with a sentinel first; the obs rows and the raw
    reward rows are followed by one more sentinel row.  raw_width: the reward_raw row stride (default 5 with the power term, 4
    without).  Returns CPU tensors of every env, and the row width."""
    from pulse_b200.humanoid_im import HumanoidImCompute
    dev = _dev()
    n = inp["body"].shape[0]
    if track is not None:
        cfg.track_body_ids, cfg.obs_version = list(track[1]), track[0]
    comp = HumanoidImCompute(ml, cfg)
    comp.termination_distances = cfg.term.to(dev).contiguous()
    comp.reset_body_mask = cfg.mask
    width = comp.obs_size
    full = torch.full((n, bodies, 13), 7.0, device=dev)
    full[:, :24] = inp["body"].to(dev)
    dof_state = torch.full((n, 72, 2), 5.0, device=dev)
    dof_state[:, :69, 1] = inp["dof_vel"].to(dev)
    dof_vel = dof_state[:, :69, 1] if interleaved else inp["dof_vel"].to(dev).contiguous()
    power = inp["dof_force"] is not None
    raw_store = torch.full((n + 1, raw_width or (5 if power else 4)), SENT, device=dev)
    obs_store = torch.full((n + 1, obs_stride or width), SENT, device=dev)
    progress = inp["progress"].to(dev).clone()
    out = {"obs_buf": obs_store[:n], "self_obs_buf": torch.full((n, 358), SENT, device=dev),
           "rew_buf": torch.full((n,), SENT, device=dev), "reward_raw": raw_store[:n],
           "reset_buf": torch.full((n,), -1, dtype=torch.long, device=dev), "terminate_buf": torch.full((n,), -1, dtype=torch.long, device=dev),
           "pass_time": torch.full((n,), 7, dtype=torch.uint8, device=dev), "fdones_out": torch.full((n,), SENT, device=dev),
           "ref_body_pos": torch.full((n, 24, 3), SENT, device=dev), "ref_body_vel": torch.full((n, 24, 3), SENT, device=dev),
           "ref_body_rot": torch.full((n, 24, 4), SENT, device=dev), "ref_dof_pos": torch.full((n, 69), SENT, device=dev)}
    rec = inp["recovery"].to(dev) if inp["recovery"] is not None else None
    comp.step(body_state=full, dof_vel=dof_vel, dof_force=inp["dof_force"].to(dev) if power else None, progress_buf=progress,
              motion_ids=inp["motion_ids"].to(dev), motion_start_times=inp["start"].to(dev), motion_start_offset=inp["offset"].to(dev),
              global_offset=inp["goff"].to(dev).contiguous(), cycle_counter=inp["cycle"].to(dev), recovery_counter=rec,
              env_ids=None if env_ids is None else env_ids.to(dev), env_count=None if env_count is None else env_count.to(dev),
              flags=inp["flags"] & 7, advance=bool(inp["flags"] & sf.ADVANCE), **out)
    torch.cuda.synchronize()
    got = {k: v.cpu() for k, v in out.items()}
    got["progress"], got["raw_tail"], got["obs_tail"] = progress.cpu(), raw_store[n].cpu(), obs_store[n].cpu()
    return got, width


def _sub(inp, sel):
    return {k: (v[sel] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == inp["body"].shape[0] else v) for k, v in inp.items()}


def check_rows(rep, tag, tb, cfg, inp, got, width, rows, track=None):
    """The written rows `rows` (env indices, ascending or not) against im_step_ref on those envs; every other row and every float past
    the row left as they were."""
    flags = inp["flags"]
    n = inp["body"].shape[0]
    sub = _sub(inp, rows)
    ref = sf.im_step_ref(table_dict(tb), sub, cfg)
    g = {"obs": got["obs_buf"][rows], "self_obs": got["self_obs_buf"][rows], "rew": got["rew_buf"][rows], "raw": got["reward_raw"][rows],
         "reset": got["reset_buf"][rows], "terminate": got["terminate_buf"][rows], "pass_time": got["pass_time"][rows],
         "progress": got["progress"][rows], "fdones": got["fdones_out"][rows]}
    if flags & sf.OBS:
        g.update(ref_body_pos=got["ref_body_pos"][rows], ref_body_vel=got["ref_body_vel"][rows], ref_body_rot=got["ref_body_rot"][rows],
                 ref_dof_pos=got["ref_dof_pos"][rows])
    sf.check_im_step(rep, tag, g, ref, flags, track=track, built=rows < BUILT)
    other = torch.ones(n, dtype=torch.bool)
    other[rows] = False
    untouched = {"obs_buf": SENT, "self_obs_buf": SENT, "rew_buf": SENT, "reward_raw": SENT, "reset_buf": -1, "terminate_buf": -1,
                 "pass_time": 7, "fdones_out": SENT, "ref_body_pos": SENT, "ref_body_vel": SENT, "ref_body_rot": SENT, "ref_dof_pos": SENT}
    for k, s in untouched.items():
        assert bool((got[k][other] == s).all()), f"{tag}: {k} written outside the env list"
    assert bool((got["obs_buf"][:, width:] == SENT).all()) and bool((got["obs_tail"] == SENT).all()), f"{tag}: obs written past the row"
    assert bool((got["raw_tail"] == SENT).all()), f"{tag}: reward_raw written past its stride"
    raw_cols = len(ref["raw"]) if flags & sf.REW else 0
    assert bool((got["reward_raw"][:, raw_cols:] == SENT).all()), f"{tag}: reward_raw written past column {raw_cols}"
    if not flags & sf.OBS:
        assert bool((got["obs_buf"] == SENT).all()) and bool((got["ref_dof_pos"] == SENT).all())
    if not flags & sf.REW:
        assert bool((got["rew_buf"] == SENT).all())
    if not flags & sf.RST:
        assert bool((got["reset_buf"] == -1).all()) and bool((got["fdones_out"] == SENT).all())
    if not flags & (sf.REW | sf.RST):
        assert bool((got["pass_time"] == 7).all())
    return ref


def _case(n, fps=30.0, flags=7, power=True, recovery=True, seed=3, **kw):
    cfg = config(**kw)
    tb = im_tables(max(40, min(n // 8, 600)), seed=4, fps=fps)
    return tb, cfg, im_inputs(tb, n, seed=seed, cfg=cfg, flags=flags, power=power, recovery=recovery)


# ---------------------------------------------------------------------------------------------------------------- the fused step
@pytest.mark.parametrize("fps", [30.0, MIXED_RATES], ids=["30fps", "mixed-fps"])
@pytest.mark.parametrize("n", [1, 7, 257, 4099, 16384])
def test_im_step_links(n, fps):
    tb, cfg, inp = _case(n, fps)
    got, width = run_step(_mlib(tb), cfg, inp)
    rep = sf.Report(f"im step n={n} fps={fps}")
    ref = check_rows(rep, "im", tb, cfg, inp, got, width, torch.arange(n))
    print("\n" + rep.text() + f"\n  rows needing four distinct frame records (one read from global memory): {ref['four']} of {n}")
    if fps != 30.0 and n >= 257:
        assert ref["four"] > 0
    if n >= BUILT:
        assert got["terminate_buf"][[18, 19]].tolist() == [0, 1]


@pytest.mark.parametrize("obs_stride,bodies,interleaved", [(941, 25, True), (934, 25, False), (941, 24, False), (936, 27, True)],
                         ids=["stride941-b25", "stride934-b25-contig", "stride941-contig", "stride936-b27"])
def test_im_step_layouts(obs_stride, bodies, interleaved):
    """obs stride 941: rows start in all four 16-byte phases (phase 3 is stored straight to global memory); 25 or 27 bodies per env:
    odd envs' body rows are only 4-byte aligned and take the non-bulk path; dof velocities strided or contiguous."""
    tb, cfg, inp = _case(4099, MIXED_RATES)
    got, width = run_step(_mlib(tb), cfg, inp, bodies=bodies, obs_stride=obs_stride, interleaved=interleaved)
    rep = sf.Report(f"im step layout {obs_stride} / {bodies}")
    check_rows(rep, "im", tb, cfg, inp, got, width, torch.arange(4099))
    print("\n" + rep.text())


FLAG_CASES = {"reward": dict(flags=1), "reset+obs": dict(flags=6), "obs": dict(flags=4), "all+advance": dict(flags=7 | sf.ADVANCE),
              "all+advance no recovery": dict(flags=7 | sf.ADVANCE, recovery=False), "reward+reset+advance": dict(flags=3 | sf.ADVANCE)}


@pytest.mark.parametrize("case", list(FLAG_CASES))
def test_im_step_flags(case):
    tb, cfg, inp = _case(257, MIXED_RATES, **FLAG_CASES[case])
    got, width = run_step(_mlib(tb), cfg, inp)
    rep = sf.Report(f"im step flags {case}")
    check_rows(rep, "im", tb, cfg, inp, got, width, torch.arange(257))
    print("\n" + rep.text())


@pytest.mark.parametrize("count", [None, 0, 60, 500, -3])
def test_im_step_env_list(count):
    """An env_ids list (permuted, with the built rows) limited by a device-side env_count: equal to 0, smaller or larger than the
    list, negative; rows outside the counted prefix stay untouched."""
    tb, cfg, inp = _case(257, MIXED_RATES, flags=7 | sf.ADVANCE)
    g = torch.Generator().manual_seed(9)
    ids = torch.cat([torch.arange(0, BUILT), BUILT + torch.randperm(257 - BUILT, generator=g)[:76]])[torch.randperm(100, generator=g)]
    cnt = None if count is None else torch.tensor([count], dtype=torch.int32)
    got, width = run_step(_mlib(tb), cfg, inp, env_ids=ids, env_count=cnt)
    c = 100 if count is None else max(0, min(count, 100))
    rows = ids[:c]
    progress_untouched = torch.ones(257, dtype=torch.bool)
    progress_untouched[rows] = False
    assert torch.equal(got["progress"][progress_untouched], inp["progress"][progress_untouched])
    rep = sf.Report(f"im step env list count={count}")
    if c:
        check_rows(rep, "im", tb, cfg, inp, got, width, rows)
    else:
        assert bool((got["obs_buf"] == SENT).all()) and bool((got["reset_buf"] == -1).all())
    print("\n" + rep.text())


CONFIGS = {"no power": dict(power=False), "no power raw stride 5": dict(power=False, raw_width=5), "cycle motion": dict(cycle_motion=True, max_episode_length=30),
           "no early termination": dict(enable_early_termination=False),
           "mean reset": dict(use_mean_reset=True, mask=mask_of(DEFAULT_RESET_BODIES[1:]), term=nonuniform_term()),
           "per-body distances": dict(term=nonuniform_term())}


@pytest.mark.parametrize("case", list(CONFIGS))
def test_im_step_configs(case):
    kw = dict(CONFIGS[case])
    raw_width = kw.pop("raw_width", None)
    tb, cfg, inp = _case(4099, 30.0, **kw)
    got, width = run_step(_mlib(tb), cfg, inp, raw_width=raw_width)
    rep = sf.Report(f"im step {case}")
    check_rows(rep, "im", tb, cfg, inp, got, width, torch.arange(4099))
    print("\n" + rep.text())
    if case != "no early termination":
        assert 0 < int(got["terminate_buf"].sum()) < 4099


# ---------------------------------------------------------------------------------------------------------------- the tracked step
TRACKS = {1: (11,), 3: (13, 2, 7), 24: tuple(int(j) for j in torch.randperm(24, generator=torch.Generator().manual_seed(2)))}


@pytest.mark.parametrize("K", [1, 3, 24])
@pytest.mark.parametrize("version", [6, 7])
def test_im_track_step_links(version, K):
    """pulse_im_track_step: the tracked row is the v6 block's columns humanoid_im.track_columns selects (ranks permuted).  v7 rows are
    packed at stride = width = 358 + 9 K, odd for odd K, so consecutive rows start in every 16-byte phase (phase 3 stored straight to
    global memory); v6 rows (358 + 24 K, phases 0 and 2) get a stride of width + 3 and sentinels between the rows."""
    tb, cfg, inp = _case(4099, MIXED_RATES)
    track = (version, TRACKS[K])
    width = 358 + (24 if version == 6 else 9) * K
    got, w = run_step(_mlib(tb), cfg, inp, obs_stride=width if version == 7 else width + 3, track=track)
    assert w == width
    rep = sf.Report(f"im track step v{version} K={K}")
    check_rows(rep, "im", tb, cfg, inp, got, w, torch.arange(4099), track=track)
    print("\n" + rep.text())


# ---------------------------------------------------------------------------------------------------------------- task observation
@pytest.mark.parametrize("upright", [True, False])
@pytest.mark.parametrize("case", TASK_CASES, ids=[f"v{c[0]}-T{c[1]}-J{len(c[2])}" for c in TASK_CASES])
def test_task_obs_links(case, upright):
    from pulse_b200 import _lib
    version, T, ids = case
    lib = _lib.load()
    dev = _dev()
    n = 4099
    body, rp, rq, rv, rw, dof, rdof = task_obs_inputs(n, T, seed=version + 10 * T)
    full = torch.full((n, 26, 13), 3.0, device=dev)
    full[:, :24] = body.to(dev)
    dof_state = torch.zeros(n, 69, 2, device=dev)
    dof_state[:, :, 0] = dof.to(dev)
    d = {k: x.to(dev).contiguous() for k, x in (("rp", rp), ("rq", rq), ("rv", rv), ("rw", rw), ("rdof", rdof))}
    tr = torch.tensor(ids, dtype=torch.int32, device=dev)
    size = lib.pulse_task_obs_size(version, len(ids), T)
    assert size == sf.task_obs_size(version, len(ids), T)
    obs = torch.full((n, size + 5), -7.0, device=dev)
    a = _lib.TaskObsArgs(body_state=full.data_ptr(), body_env_stride=full.stride(0), track_ids=tr.data_ptr(), num_track=len(ids), time_steps=T,
                         version=version, upright=int(upright), ref_pos=d["rp"].data_ptr(), ref_rot=d["rq"].data_ptr(), ref_vel=d["rv"].data_ptr(),
                         ref_ang_vel=d["rw"].data_ptr(), dof_pos=dof_state.data_ptr(), dof_env_stride=dof_state.stride(0), dof_elem_stride=2,
                         ref_dof_pos=d["rdof"].data_ptr(), obs=obs.data_ptr(), obs_stride=obs.stride(0), num_envs=n)
    _lib.check(lib.pulse_im_task_obs(C.byref(a), _lib.current_stream(dev)), "pulse_im_task_obs")
    torch.cuda.synchronize()
    o = obs.cpu()
    assert bool((o[:, size:] == -7.0).all())
    rep = sf.Report(f"task obs v{version} T={T} J={len(ids)} upright={upright}")
    ref = sf.task_obs_ref(version, T, ids, upright, body, rp, rq, rv, rw, dof, rdof)
    sf.check_task_obs(rep, "task", o, ref, built=torch.arange(n) < 2)
    print("\n" + rep.text())
