"""Per-step env reset (SURVEY rows a13 / 8f-3) through `pulse_reset_ref_state` + the observation-mode step kernel, against the
oracle's restatement of the reference's reset chain (`oracle.pulse_oracle.reset_envs`: humanoid.py:574-609,
humanoid_amp.py:468-488, :519-597, humanoid_im.py:921-989, motion_lib_base.py:411-420).

Bars: env list / actor list / count and every integer buffer bit-exact; simulator tensors, AMP rows and observations within 1e-4
(rtol for the exponential-map dof positions, see test_gpu_step._check_step); buffers of envs that are NOT reset bit-identical."""
import pytest
import torch

from tests.helpers import exact_step_inputs, exact_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ATOL = 1e-4


def _setup(n, clips=37, seed=3, fps=30.0):
    from oracle import pulse_oracle as po
    from pulse_b200.humanoid_im import HumanoidImCompute
    from pulse_b200.motion_lib import MotionLibB200
    tb = exact_tables(clips, seed=seed, fps=fps)
    z, _ = exact_step_inputs(tb, n, seed=seed + 1)
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames", "dt",
                                                                 "length_starts")}, device=DEV)
    comp = HumanoidImCompute(ml)
    g = torch.Generator().manual_seed(seed + 2)
    st = {  # oracle-side state (dense CPU tensors)
        "motion_ids": z["motion_ids"], "start_times": z["start_times"], "start_offset": 0.01 * torch.randn(n, generator=g),
        "global_offset": z["global_offset"], "cycle_counter": z["cycle_counter"], "progress_buf": z["progress_buf"],
        "reset_buf": torch.zeros(n, dtype=torch.long), "terminate_buf": (torch.rand(n, generator=g) < 0.3).long(),
        "root_states": torch.randn(n, 13, generator=g), "dof_pos": z["dof_pos"], "dof_vel": z["dof_vel"], "body_state": z["body_state"],
        "contact_forces": torch.randn(n, 24, 3, generator=g), "amp_obs_buf": torch.randn(n, 10, 196, generator=g),
        "obs_buf": torch.randn(n, 934, generator=g), "dof_force": z["dof_force"],
    }
    return po, tb, comp, st, g


def _device_state(st, n):
    """Isaac-Gym shaped device tensors: 2 actors per env in the root tensor, 72 dofs x (pos, vel), 26 bodies."""
    d = {k: v.to(DEV).clone() for k, v in st.items() if k not in ("root_states", "dof_pos", "dof_vel", "body_state", "contact_forces")}
    root_all = torch.full((n, 2, 13), 5.0, device=DEV)
    root_all[:, 0] = st["root_states"].to(DEV)
    dof_state = torch.full((n, 72, 2), 5.0, device=DEV)
    dof_state[:, :69, 0], dof_state[:, :69, 1] = st["dof_pos"].to(DEV), st["dof_vel"].to(DEV)
    body = torch.full((n, 26, 13), 5.0, device=DEV)
    body[:, :24] = st["body_state"].to(DEV)
    contact = torch.full((n, 26, 3), 5.0, device=DEV)
    contact[:, :24] = st["contact_forces"].to(DEV)
    d.update(root_all=root_all, dof_state=dof_state, body=body, contact=contact,
             actor_ids=(torch.arange(n, dtype=torch.int32, device=DEV) * 2))
    return d


def _call(comp, d, phase=None, env_ids=None, **kw):
    return comp.reset_envs(motion_ids=d["motion_ids"], motion_start_times=d["start_times"], motion_start_offset=d["start_offset"],
                           global_offset=d["global_offset"], progress_buf=d["progress_buf"], root_states=d["root_all"][:, 0],
                           dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1], rigid_body_state=d["body"],
                           reset_buf=None if env_ids is not None else d["reset_buf"], env_ids=env_ids, terminate_buf=d["terminate_buf"],
                           cycle_counter=d["cycle_counter"], contact_forces=d["contact"], amp_obs_buf=d["amp_obs_buf"], actor_ids=d["actor_ids"],
                           phase=phase, obs_buf=d["obs_buf"], **kw)


def _compare(d, exp, ids, n):
    close = lambda a, b, **k: torch.testing.assert_close(a.cpu(), b, **({"atol": ATOL, "rtol": 0} | k))
    for k in ("progress_buf", "reset_buf", "terminate_buf", "cycle_counter"):
        assert torch.equal(d[k].cpu(), exp[k]), k
    assert torch.equal(d["start_times"].cpu(), exp["start_times"])          # the start time is index arithmetic: bit-exact
    assert torch.equal(d["start_offset"].cpu(), exp["start_offset"]) and torch.equal(d["global_offset"].cpu(), exp["global_offset"])
    close(d["root_all"][:, 0], exp["root_states"], atol=1e-5)
    close(d["dof_state"][:, :69, 0], exp["dof_pos"], rtol=1e-4)
    close(d["dof_state"][:, :69, 1], exp["dof_vel"], atol=1e-5)
    close(d["body"][:, :24], exp["body_state"], atol=1e-5)
    close(d["contact"][:, :24], exp["contact_forces"], atol=0)
    close(d["amp_obs_buf"], exp["amp_obs_buf"])
    close(d["obs_buf"], exp["obs_buf"])
    # padding (second actor, extra dofs / bodies) and every env that was not reset: untouched bit for bit
    assert float((d["root_all"][:, 1] - 5.0).abs().max()) == 0 and float((d["dof_state"][:, 69:] - 5.0).abs().max()) == 0
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids] = False
    # `_contact_forces[env_ids] = 0` (humanoid.py:606) clears EVERY body row of a reset env, the non-humanoid ones included
    assert float((d["body"][:, 24:] - 5.0).abs().max()) == 0 and float((d["contact"][keep, 24:] - 5.0).abs().max() if keep.any() else 0) == 0
    assert float(d["contact"][ids].abs().max()) == 0
    for ours, ref in ((d["root_all"][:, 0], exp["root_states"]), (d["body"][:, :24], exp["body_state"]), (d["amp_obs_buf"], exp["amp_obs_buf"]),
                      (d["obs_buf"], exp["obs_buf"]), (d["dof_state"][:, :69, 0], exp["dof_pos"])):
        assert torch.equal(ours.cpu()[keep], ref[keep])


@pytest.mark.parametrize("n,frac,fps", [pytest.param(300, 0.12, 30.0, id="300-0.12"), pytest.param(2051, 0.05, 30.0, id="2051-0.05"),
                                        pytest.param(64, 1.0, 30.0, id="64-1.0"),
                                        pytest.param(2051, 0.3, (24.0, 25.0, 29.97, 50.0, 60.0, 120.0), id="2051-0.3-mixed-fps")])
def test_reset_envs_mask_mode_matches_oracle(n, frac, fps):
    """Mixed rates run the reset kernels' own frame blend and slerp (reset_state.cuh) on clips off 30 fps, the AMP history rows included."""
    po, tb, comp, st, g = _setup(n, fps=fps)
    mask = (torch.rand(n, generator=g) < frac)
    mask[0] = mask[n - 1] = True
    st["reset_buf"] = mask.long() * 3                      # any non-zero value marks a reset
    phase = torch.rand(n, generator=g)
    d = _device_state(st, n)
    ws = _call(comp, d, phase=phase.to(DEV))
    ids = mask.nonzero().flatten()
    torch.cuda.synchronize()
    cnt = int(ws["count"].item())
    assert cnt == ids.numel()
    assert torch.equal(ws["env_list"][:cnt].cpu(), ids) and torch.equal(ws["actor_list"][:cnt].cpu(), (ids * 2).int())
    exp = po.reset_envs(tb, po.ImStepConfig(), st, ids, phase)
    _compare(d, exp, ids, n)


def test_reset_envs_list_mode_and_empty():
    n = 130
    po, tb, comp, st, g = _setup(n, seed=9)
    phase = torch.rand(n, generator=g)
    ids = torch.tensor([2, 3, 64, 65, 129])
    d = _device_state(st, n)
    ws = _call(comp, d, phase=phase.to(DEV), env_ids=ids.to(DEV))
    torch.cuda.synchronize()
    assert int(ws["count"].item()) == 5 and torch.equal(ws["env_list"][:5].cpu(), ids)
    _compare(d, po.reset_envs(tb, po.ImStepConfig(), st, ids, phase), ids, n)
    # nothing to reset: no buffer changes, count 0
    d2 = _device_state(st, n)
    before = {k: v.clone() for k, v in d2.items()}
    ws = _call(comp, d2, phase=phase.to(DEV))
    torch.cuda.synchronize()
    assert int(ws["count"].item()) == 0
    for k, v in d2.items():
        assert torch.equal(v, before[k]), k


def test_reset_envs_philox_draws():
    """Without injected draws the start times come from Philox4x32-10 inside the kernel: on the reference's 1/30 s grid, inside the
    clip, reproducible for (seed, offset), different across offsets, and spread over the clip."""
    n = 4096
    po, tb, comp, st, g = _setup(n, clips=64, seed=21)
    st["reset_buf"] = torch.ones(n, dtype=torch.long)
    runs = []
    for off in (0, 0, 1):
        d = _device_state(st, n)
        _call(comp, d, seed=1234, offset=off)
        torch.cuda.synchronize()
        runs.append(d["start_times"].cpu())
    assert torch.equal(runs[0], runs[1]) and not torch.equal(runs[0], runs[2])
    t = runs[0]
    L = tb.lengths[st["motion_ids"]]
    k = torch.round(t.double() * 30)
    assert torch.equal((k * (1 / 30)).float(), t) or float((t - (k.float() * (1 / 30))).abs().max()) < 1e-6
    assert bool((t >= 0).all()) and bool((t <= L + 1e-6).all())
    u = (t / L.clamp(min=1e-6))[L > 1.0]
    assert 0.40 < float(u.mean()) < 0.60 and float(u.std()) > 0.2
