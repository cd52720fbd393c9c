"""The tracked-body imitation step (`pulse_im_track_step`) and the VR controller task's rollout driver (`ImZStepsB200`).

Bars: the tracked step bit for bit against `pulse_im_step` on the same inputs (self columns, reward, raw reward, reset, terminate, dones,
counters, side buffers; each task column equal to the column-map gather of the full 934-float row), over v6 / v7, sorted, unsorted and
single-body lists, all 24 bodies, a v7 stride with rows 3 floats past a 16-byte boundary and PULSE_STEP_ADVANCE; the task block within
1e-4 of the general task-observation kernel; list mode after `pulse_reset_ref_state`; the driver's graph-captured horizon bit for bit
against its sequential schedule, hook mode as graph segments, the Philox blocks `philox_blocks` names regenerated on the host against
the kernels' draws, `mus` against `act()`, and `finish` / `train_epoch` over the 6-layer policy.  Fixtures are seeded synthetic state."""
import pytest
import torch

from tests.helpers import exact_step_inputs, exact_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIPS = 29
VR = (13, 18, 23)
UNITS = (2048, 1536, 1024, 1024, 512, 512)     # pulse_z_vr.yaml


def _motion_lib(fps):
    from pulse_b200.motion_lib import MotionLibB200
    tb = exact_tables(CLIPS, seed=13, fps=fps)
    return MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames",
                                                                   "dt", "length_starts")}, device=DEV), tb


@pytest.fixture(scope="module")
def ml():
    return _motion_lib(30.0)


@pytest.fixture(scope="module")
def ml_mixed_fps():
    """Clips at 24 to 120 fps: above 30 fps the step reads a fourth frame row straight from the records."""
    return _motion_lib((24.0, 25.0, 29.97, 30.0, 50.0, 60.0, 120.0))


def _sim(tb, n, seed):
    """Isaac-Gym shaped state (2 actors per env, 72 dofs x (pos, vel), 26 bodies) near the reference frames; every 7th env is displaced
    by 1 m (early termination), every 11th is past the end of its clip."""
    z, _ = exact_step_inputs(tb, n, seed=seed)
    body = torch.zeros(n, 26, 13)
    body[:, :24] = z["body_state"]
    body[::7, :24, 0:3] += 1.0
    progress = z["progress_buf"].clone()
    progress[::7] = progress[::7].clamp(min=2)
    progress[::11] = 2000
    root = torch.zeros(n, 2, 13)
    root[:, 0] = body[:, 0]
    root[:, 1, 6] = 1.0
    dof = torch.zeros(n, 72, 2)
    dof[:, :69, 0], dof[:, :69, 1] = z["dof_pos"], z["dof_vel"]
    g = torch.Generator().manual_seed(seed + 1)
    sim = dict(body_state=body, root_all=root, dof_state=dof, progress_buf=progress, motion_ids=z["motion_ids"].clone(),
               motion_start_times=z["start_times"].clone(), motion_start_offset=0.01 * torch.randn(n, generator=g),
               global_offset=z["global_offset"].clone(), dof_force=z["dof_force"], contact_forces=torch.randn(n, 26, 3, generator=g),
               actor_ids=torch.arange(n, dtype=torch.int32) * 2)
    sim = {k: v.to(DEV) for k, v in sim.items()}
    sim.update(root_states=sim["root_all"][:, 0], dof_pos=sim["dof_state"][:, :69, 0], dof_vel=sim["dof_state"][:, :69, 1])
    return sim


def _kw(s):
    return {k: s[k] for k in ("body_state", "progress_buf", "motion_ids", "motion_start_times", "motion_start_offset", "global_offset")}


def _outs(n, width, stride):
    return dict(obs=torch.full((n, stride), 7.5, device=DEV), rew=torch.zeros(n, device=DEV), raw=torch.zeros(n, 5, device=DEV),
                reset=torch.zeros(n, dtype=torch.long, device=DEV), term=torch.zeros(n, dtype=torch.long, device=DEV),
                dones=torch.full((n,), 3.0, device=DEV), rbp=torch.zeros(n, 24, 3, device=DEV), rbr=torch.zeros(n, 24, 4, device=DEV),
                rbv=torch.zeros(n, 24, 3, device=DEV), prog=None)


def _run(comp, s, o, flags, advance):
    from pulse_b200 import _lib  # noqa: F401
    kw = _kw(s)
    kw["progress_buf"] = o["prog"] = s["progress_buf"].clone()
    comp.step(flags=flags, advance=advance, obs_buf=o["obs"], rew_buf=o["rew"], reward_raw=o["raw"], reset_buf=o["reset"], terminate_buf=o["term"],
              fdones_out=o["dones"], dof_force=s["dof_force"], dof_vel=s["dof_vel"], ref_body_pos=o["rbp"], ref_body_rot=o["rbr"],
              ref_body_vel=o["rbv"], **kw)


# ------------------------------------------------------------------------------------------------ 1. the tracked step vs the full row
@pytest.mark.parametrize("ids,version,pad,advance,fast", [
    (VR, 6, 0, False, False), (VR, 7, 0, False, False), ((23, 5, 13, 0, 18), 6, 3, False, False), (tuple(range(24)), 6, 0, False, False),
    ((7,), 7, 0, False, False), (VR, 6, 5, True, False), ((18, 13), 7, 1, True, False), ((23, 5, 13, 0, 18), 6, 0, False, True),
    (tuple(range(23)), 6, 0, False, True)])
def test_track_step_equals_full_row_gather(ml, ids, version, pad, advance, fast):
    """v7 over 3 bodies is 385 floats wide and (7,) 367: a dense [N, W] buffer then has every fourth row 3 floats past a 16-byte
    boundary, the rows the kernel stores directly.  `fast`: body velocities 30 times larger (differences well above 8 m/s and rad/s,
    where one rounding exceeds 1e-6).  23 bodies: the widest row beside the 24-float sink of the untracked body."""
    _track_vs_full(ml, ids, version, pad, advance, fast)


@pytest.mark.parametrize("ids,version,pad,advance,fast", [(VR, 6, 0, False, False), (VR, 7, 0, True, False), (tuple(range(24)), 6, 0, False, False),
                                                          ((23, 5, 13, 0, 18), 6, 0, False, True)])
def test_track_step_equals_full_row_gather_mixed_fps(ml_mixed_fps, ids, version, pad, advance, fast):
    _track_vs_full(ml_mixed_fps, ids, version, pad, advance, fast)


def _track_vs_full(ml, ids, version, pad, advance, fast):
    from pulse_b200 import _lib
    from pulse_b200.humanoid_im import SELF_OBS, HumanoidImCompute, ImConfig, track_columns
    lib, tb = ml
    n = 1027
    s = _sim(tb, n, seed=31)
    if fast:
        s["body_state"][..., 7:13] *= 30.0
    full, tr = HumanoidImCompute(lib), HumanoidImCompute(lib, ImConfig(track_body_ids=ids, obs_version=version))
    W = tr.obs_size
    a, b = _outs(n, 934, 934), _outs(n, W, W + pad)
    _run(full, s, a, _lib.STEP_ALL, advance)
    _run(tr, s, b, _lib.STEP_ALL, advance)
    if W % 4 == 1 and pad == 0:
        assert {(r * W) % 4 for r in range(4)} == {0, 1, 2, 3}
    assert torch.equal(b["obs"][:, :SELF_OBS], a["obs"][:, :SELF_OBS])
    got, want = b["obs"][:, SELF_OBS:W], a["obs"][:, SELF_OBS:][:, track_columns(version, ids).to(DEV)]
    assert torch.equal(got, want), (int((got != want).sum()), float((got - want).abs().max()))
    assert float((b["obs"][:, W:] - 7.5).abs().max()) == 0 if pad else True
    if len(ids) == 24 and version == 6:                            # the whole 934-float row
        assert torch.equal(b["obs"], a["obs"])
    for k in ("rew", "raw", "reset", "term", "dones", "prog", "rbp", "rbr", "rbv"):
        assert torch.equal(a[k], b[k]), k
    assert 0 < int(a["reset"].sum()) < n and 0 < int(a["term"].sum()) and bool((a["term"][::7] == 1).all())
    assert torch.equal(a["prog"], s["progress_buf"] + (1 if advance else 0))


def test_task_block_matches_general_kernel(ml):
    """The tracked task block against `HumanoidImCompute.task_obs` (the general kernel behind the three-launch path, pinned to the
    reference's goldens) on the same state, within 1e-4."""
    from pulse_b200 import _lib
    from pulse_b200.humanoid_im import SELF_OBS, HumanoidImCompute, ImConfig
    lib, tb = ml
    n = 1027
    s = _sim(tb, n, seed=37)
    for ids, version in ((VR, 6), (VR, 7), ((23, 5, 13, 0, 18), 6)):
        tr = HumanoidImCompute(lib, ImConfig(track_body_ids=ids, obs_version=version))
        W = tr.obs_size
        obs = torch.zeros(n, W, device=DEV)
        tr.step(flags=_lib.STEP_OBS, obs_buf=obs, **_kw(s))
        task = torch.zeros(n, W - SELF_OBS, device=DEV)
        tr.task_obs(version=version, track_ids=torch.tensor(ids, dtype=torch.int32, device=DEV), obs_buf=task, **_kw(s))
        torch.testing.assert_close(obs[:, SELF_OBS:], task, atol=1e-4, rtol=0)


def test_list_mode_after_reset(ml):
    """`reset_envs(obs_buf=...)` in mask mode writes the tracked rows of the reset envs only (device-side count): they equal an all-env
    observation call on the reset state, the other rows keep a sentinel."""
    from pulse_b200 import _lib
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    lib, tb = ml
    n = 1027
    s = _sim(tb, n, seed=41)
    tr = HumanoidImCompute(lib, ImConfig(track_body_ids=VR))
    reset = torch.zeros(n, dtype=torch.long, device=DEV)
    reset[::5] = 1
    reset[n - 1] = 1
    ids = reset.nonzero().flatten()
    obs = torch.full((n, 430), -3.25, device=DEV)
    ws = tr.reset_envs(motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"], motion_start_offset=s["motion_start_offset"],
                       global_offset=s["global_offset"], progress_buf=s["progress_buf"], root_states=s["root_states"], dof_pos=s["dof_pos"],
                       dof_vel=s["dof_vel"], rigid_body_state=s["body_state"], reset_buf=reset, phase=torch.rand(n, device=DEV), obs_buf=obs)
    assert int(ws["count"]) == ids.numel()
    ref = torch.zeros(n, 430, device=DEV)
    tr.step(flags=_lib.STEP_OBS, obs_buf=ref, **_kw(s))
    assert torch.equal(obs[ids], ref[ids])
    keep = torch.ones(n, dtype=torch.bool, device=DEV)
    keep[ids] = False
    assert float((obs[keep] + 3.25).abs().max()) == 0


# ------------------------------------------------------------------------------------------------ 2. the driver
def _policy(seed=0, units=(256, 128)):
    from pulse_b200.ppo import PPOPolicy
    pol = PPOPolicy(obs_size=430, num_actions=32, units=units, act="silu", logstd=-1.5, device=DEV, seed=seed)
    g = torch.Generator().manual_seed(seed + 40)
    pol.obs_rms.running_mean.copy_(0.1 * torch.randn(pol.obs_size, generator=g, dtype=torch.float64))
    pol.obs_rms.running_var.copy_(0.5 + torch.rand(pol.obs_size, generator=g, dtype=torch.float64))
    pol.obs_rms._refresh()
    pol.value_rms.running_mean.fill_(0.7)
    pol.value_rms.running_var.fill_(2.3)
    pol.value_rms._refresh()
    return pol


def _driver(ml, n, T=4, seed=5, use_graphs=True, units=(256, 128)):
    from pulse_b200.humanoid_im import HumanoidImCompute, ImConfig
    from pulse_b200.imz_rollout import ImZStepsB200
    from pulse_b200.vae import PulseVAE
    lib, tb = ml
    comp = HumanoidImCompute(lib, ImConfig(track_body_ids=VR))
    g = torch.Generator().manual_seed(seed + 1)
    freeze = torch.zeros(69, dtype=torch.uint8)
    freeze[[9, 10, 11, 66, 67, 68]] = 1
    drv = ImZStepsB200(comp, _policy(units=units), PulseVAE(device=DEV, with_critic=False, seed=1), _sim(tb, n, seed), horizon=T,
                       pd_offset=torch.randn(69, generator=g).to(DEV), pd_scale=(0.5 + torch.rand(69, generator=g)).to(DEV),
                       pd_freeze=freeze.to(DEV), use_graphs=use_graphs, reset_seed=3)
    drv.first_observation()
    return drv


def _state(drv):
    s = drv.sim
    out = {k: getattr(drv, k) for k in ("obses", "obs_carry", "actions", "mus", "neglogp", "values", "next_values", "rewards", "dones", "pd_tar",
                                        "reset_buf", "terminate_buf")}
    out.update({k: s[k] for k in ("body_state", "root_all", "dof_state", "contact_forces", "progress_buf", "motion_ids", "motion_start_times",
                                  "motion_start_offset", "global_offset")})
    return out


def _assert_same(a, b, what=""):
    sa, sb = _state(a), _state(b)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f"{what}: {k} differs"


@pytest.mark.parametrize("n", [1027, 3072])
def test_horizon_graph_equals_sequential(ml, n):
    T = 4
    a = _driver(ml, n, T=T, use_graphs=True)
    b = _driver(ml, n, T=T, use_graphs=False)
    _assert_same(a, b, "initial")
    for use in ("eager", "capture", "replay"):
        a.play_steps()
        b.play_steps()
        _assert_same(a, b, use)
        if use == "eager":                  # step 0 resets the displaced envs and those past the end of their clip
            assert bool((b.dones[0][::7] == 1).all()) and bool((b.dones[0][::11] == 1).all()) and float(b.dones.sum()) < T * n / 2
        a.finish()
        b.finish()
        assert torch.equal(a.adv, b.adv) and torch.equal(a.ret, b.ret)
    assert isinstance(a._graphs[("horizon",)], torch.cuda.CUDAGraph)
    assert bool(torch.isfinite(a.obses).all()) and bool(torch.isfinite(a.next_values).all())
    pol = b.policy                          # the driver's mus are the policy's act() on the observations of each step
    for t in range(T):
        assert torch.equal(pol.act(b.obses[:, t], eps=torch.zeros(n, 32, device=DEV))["mus"], b.mus[:, t]), t


def test_hooks_run_as_graph_segments(ml):
    n, T = 1027, 3
    a = _driver(ml, n, T=T, use_graphs=True)
    b = _driver(ml, n, T=T, use_graphs=False)

    def physics_of(drv):
        noise = torch.zeros(n, 26, 3, device=DEV)

        def physics(t):                     # a deterministic stand-in for the simulator: perturbs the body positions
            noise.copy_(0.02 * torch.randn(n, 26, 3, generator=torch.Generator().manual_seed(100 + t)))
            drv.sim["body_state"][..., 0:3].add_(noise)
            drv.sim["root_all"][:, 0, 0:3].add_(noise[:, 0])
        return physics

    a.physics, b.physics = physics_of(a), physics_of(b)
    counts = []
    a.refresh = lambda t, ws: counts.append(ws["count"].clone())
    b.refresh = lambda t, ws: None
    for use in ("eager", "capture", "replay"):
        a.play_steps()
        b.play_steps()
        _assert_same(a, b, use)
    assert sum(int(c) for c in counts) > 0
    assert all(isinstance(a._graphs[(seg, t)], torch.cuda.CUDAGraph) for seg in ("reset", "act", "post") for t in range(T))


def test_philox_blocks_are_the_kernels_draws(ml):
    """`philox_blocks` names the blocks the kernels read: the start-time uniforms regenerated on the host and injected reproduce the
    driver's reset bit for bit; the latent noise the driver drew equals the host's Box-Muller of the named blocks (within the tolerance
    of the kernel's __logf / __sincosf)."""
    import numpy as np

    from pulse_b200.imz_rollout import philox_blocks
    from tests.philox_ref import box_muller, philox4x32_10, u01
    n, t, off = 1027, 3, 64
    a = _driver(ml, n, use_graphs=False)
    b = _driver(ml, n, use_graphs=False)
    for d in (a, b):
        d.policy.rng_offset.fill_(off)
        d.reset_buf[::3] = 1
    a._reset(t)
    a._reset_obs(t)
    blocks = [philox_blocks(e, t, off) for e in range(n)]
    x = philox4x32_10(b.reset_seed, [bl[0][1] for bl in blocks], [bl[0][2] for bl in blocks])[0]
    s = b.sim
    b.reset_ws = b.comp.reset_envs(motion_ids=s["motion_ids"], motion_start_times=s["motion_start_times"],
                                   motion_start_offset=s["motion_start_offset"], global_offset=s["global_offset"], progress_buf=s["progress_buf"],
                                   root_states=s["root_states"], dof_pos=s["dof_pos"], dof_vel=s["dof_vel"], rigid_body_state=s["body_state"],
                                   reset_buf=b.reset_buf, contact_forces=s["contact_forces"], actor_ids=s["actor_ids"],
                                   phase=torch.from_numpy(u01(x)).to(DEV))
    b._reset_obs(t)
    _assert_same(a, b, "injected draws")
    assert int(b.reset_ws["count"]) == len(range(0, n, 3))
    a._act(t)
    pw = philox4x32_10(a.policy.rng_seed, [i for bl in blocks for _, i, _ in bl[1:]], [c for bl in blocks for _, _, c in bl[1:]])
    n0, n1 = (w.reshape(n, -1) for w in box_muller(pw[0], pw[1]))
    eps = np.empty((n, 32))
    eps[:, 0::2], eps[:, 1::2] = n0, n1
    drawn = (a.actions[:, t] - a.mus[:, t]) / torch.exp(a.policy.logstd)
    err = (drawn.double().cpu() - torch.from_numpy(eps)).abs()
    assert float(err.max()) < 2e-3 and float(err.mean()) < 2e-5, (float(err.max()), float(err.mean()))


def test_finish_and_train_epoch(ml):
    """One iteration over the 6-layer pulse_z_vr.yaml policy: `finish` and `train_epoch` run under graphs, change the weights, and a
    replayed iteration issues no host synchronisation."""
    n, T = 1024, 4
    a = _driver(ml, n, T=T, use_graphs=True, units=UNITS)
    before = a.policy.flat.params.clone()
    for _ in range(2):
        a.play_steps()
        a.finish()
        stats = a.train_epoch(mini_epochs=2, minibatch=1024)
    assert float(stats.abs().sum()) > 0 and bool(torch.isfinite(a.policy.flat.params).all())
    assert not torch.equal(before, a.policy.flat.params)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a.play_steps()
        a.finish()
        a.train_epoch(mini_epochs=2, minibatch=1024)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
