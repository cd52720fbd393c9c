"""The PULSE-X speed task on the device (52-body SMPL-X humanoid, HumanoidSpeedZ with robot=smplx_humanoid): `pulse_smplx_speed_step`,
its list observation and rollout step against the oracle restatement pinned by the reference fixture (observation and reward within
1e-5, reset and terminate bit-exact) at 1, 300, 2051 and 16384 envs; the 52-body MotionLib query; the reset `pulse_reset_ztask_smplx`
against the oracle (env list, counters and clips bit-exact, the scattered state within 1e-5); the driver's graph-captured horizon bit
for bit against the eager one with resets inside it, then `train_epoch`; `pulse_latent_post` at E = 48 against `latent_post_ref`."""
import ctypes as C

import pytest
import torch

from oracle import pulse_oracle as po
from tests import smplx_speed_oracle as so
from tests import ztask_reset_oracle as zo
from tests.test_smplx_speed_cpu import gen

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIPS = 17


def _views(z, extra=1):
    """Isaac-Gym shaped views with `extra` bodies after the humanoid's 52 (another actor's)."""
    n = z["body_state"].shape[0]
    rb = torch.full((n, so.BODIES + extra, 13), 5.0, device=DEV)
    rb[:, :so.BODIES] = z["body_state"].to(DEV)
    cf = torch.zeros(n, so.BODIES + extra, 3, device=DEV)
    cf[:, :so.BODIES] = z["contact_forces"].to(DEV)
    return rb, cf


def _task(m, n, z, contacts):
    from pulse_b200.ztasks import SmplxSpeedTaskB200
    task = SmplxSpeedTaskB200(n, DEV, contact_body_ids=contacts, max_episode_length=m.MAX_LEN, dt=m.DT)
    task._prev_root_pos.copy_(z["prev_root_pos"].to(DEV))
    task._tar_speed.copy_(z["tar_speed"].to(DEV))
    return task


def _check_rows(m, z, contacts, obs, rew, reset, term, rows=None):
    want_obs, want_rew, want_rs, want_tm = so.step(z, contacts, m.MAX_LEN, m.DT)
    if rows is not None:
        want_obs = want_obs[rows]
    torch.testing.assert_close(obs.cpu(), want_obs, atol=1e-5, rtol=0)
    if rew is not None:
        torch.testing.assert_close(rew.cpu(), want_rew, atol=1e-5, rtol=0)
        assert torch.equal(reset.cpu(), want_rs) and torch.equal(term.cpu(), want_tm)


@pytest.mark.parametrize("contact_set", ["feet", "feet_and_bodies_above_31"])
@pytest.mark.parametrize("n", [1, 300, 2051, 16384])
def test_step_list_and_rollout_rows(n, contact_set):
    """contact_set feet_and_bodies_above_31 (CONTACT_IDS_HI) pins the 64-bit contact mask: rows 2::17 fall unless body 40's bit is set."""
    from pulse_b200 import _lib
    m = gen()
    contacts = m.CONTACT_IDS if contact_set == "feet" else m.CONTACT_IDS_HI
    z = m.inputs(n, seed=n)
    rb, cf = _views(z)
    task = _task(m, n, z, contacts)
    task.post_physics_step(rb, z["progress_buf"].to(DEV), cf)
    torch.cuda.synchronize()
    _check_rows(m, z, contacts, task.obs_buf, task.rew_buf, task.reset_buf, task._terminate_buf)
    torch.testing.assert_close(task.reward_raw[:, 0], task.rew_buf, atol=0, rtol=0)
    if n > 1:
        assert int(task._terminate_buf.sum()) > 0 and int(task.reset_buf.sum()) >= int(task._terminate_buf.sum())
    # the list observation writes the listed rows and nothing else
    ids = torch.arange(0, n, 3, device=DEV)
    count = torch.tensor([ids.numel()], dtype=torch.int32, device=DEV)
    task.obs_buf.fill_(-7.0)
    task.observe_list(rb, ids, count, z["progress_buf"].to(DEV), cf)
    torch.cuda.synchronize()
    _check_rows(m, z, contacts, task.obs_buf[ids], None, None, None, rows=ids.cpu())
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids.cpu()] = False
    assert bool((task.obs_buf.cpu()[keep] == -7.0).all())
    # the rollout step: progress += 1 inside the kernel, then the step, then dones = float(reset)
    prog = (z["progress_buf"] - 1).to(DEV)
    dones = torch.full((n,), -1.0, device=DEV)
    a = task._args(rb, prog, cf)
    _lib.check(task.lib.pulse_smplx_speed_rollout_step(C.byref(a), dones.data_ptr(), n, _lib.current_stream(DEV)), "rollout")
    torch.cuda.synchronize()
    assert torch.equal(prog.cpu(), z["progress_buf"])
    _check_rows(m, z, contacts, task.obs_buf, task.rew_buf, task.reset_buf, task._terminate_buf)
    assert torch.equal(dones, task.reset_buf.float())
    pinned = torch.arange(2, max(n, 2), 17)
    pinned = pinned[z["progress_buf"][pinned] > 1]
    if pinned.numel():
        assert bool((task._terminate_buf.cpu()[pinned] == (1 if contact_set == "feet" else 0)).all())


@pytest.fixture(scope="module")
def motion():
    from pulse_b200.motion_lib import MotionLibB200
    tb = so.tables(CLIPS, seed=5)
    ml = MotionLibB200.from_tables(so.table_dict(tb), device=DEV)
    g = torch.Generator().manual_seed(3)
    floor = -0.9 + 0.05 * torch.rand(tb.gts.shape[0], generator=g)
    return tb, ml, floor


def test_motion_state_query(motion):
    tb, ml, _ = motion
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(0, CLIPS, (999,), generator=g)
    t = torch.rand(999, generator=g) * tb.lengths[ids] * 1.1
    got = ml.get_motion_state(ids.to(DEV), t.to(DEV))
    want = po.motion_state(tb, ids, t)
    assert ml.smplx and ml.num_bodies == 52
    for k in ("root_pos", "root_rot", "root_vel", "root_ang_vel", "dof_pos", "dof_vel", "rg_pos", "rb_rot", "body_vel", "body_ang_vel"):
        assert got[k].shape == want[k].shape, k
        torch.testing.assert_close(got[k].cpu(), want[k], atol=2e-5, rtol=0, msg=lambda s, k=k: f"{k}: {s}")


@pytest.mark.parametrize("state_init", ["Random", "Start"])
def test_reset_matches_oracle(motion, state_init):
    from pulse_b200.ztask_reset import ZTaskResetB200
    tb, ml, floor = motion
    n = 2051
    g = torch.Generator().manual_seed(8)
    st = dict(root_states=torch.randn(n, 13, generator=g), dof_pos=torch.randn(n, 153, generator=g), dof_vel=torch.randn(n, 153, generator=g),
              body_state=torch.randn(n, 53, 13, generator=g), sampled_motion_ids=torch.zeros(n, dtype=torch.int64), motion_start_times=torch.zeros(n),
              progress_buf=torch.randint(0, 300, (n,), generator=g), reset_buf=(torch.rand(n, generator=g) < 0.3).long(),
              terminate_buf=torch.ones(n, dtype=torch.int64), contact_forces=torch.randn(n, 53, 3, generator=g))
    motion_u, phase = torch.rand(n, generator=g), torch.rand(n, generator=g)
    d = {k: v.to(DEV) for k, v in st.items()}
    r = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False, state_init=state_init)
    ws = r.reset_envs(root_states=d["root_states"], dof_pos=d["dof_pos"], dof_vel=d["dof_vel"], rigid_body_state=d["body_state"],
                      progress_buf=d["progress_buf"], sampled_motion_ids=d["sampled_motion_ids"], motion_start_times=d["motion_start_times"],
                      reset_buf=d["reset_buf"], terminate_buf=d["terminate_buf"], contact_forces=d["contact_forces"],
                      motion_u=motion_u.to(DEV), phase=phase.to(DEV))
    torch.cuda.synchronize()
    ids = torch.nonzero(st["reset_buf"]).flatten()
    cnt = int(ws["count"].item())
    assert cnt == ids.numel() > 0 and torch.equal(ws["env_list"][:cnt].cpu(), ids)
    cdf = torch.cumsum(ml._sampling_batch_prob.cpu(), 0)
    v = torch.minimum(motion_u * cdf[-1], torch.nextafter(cdf[-1], torch.tensor(0.0)))
    clips = torch.searchsorted(cdf, v, right=True)
    assert torch.equal(d["sampled_motion_ids"].cpu()[ids], clips[ids])
    s = zo.sample_ref_state(tb, clips[ids], phase[ids], floor, zo.FACE_X, False, zo.RANDOM if state_init == "Random" else zo.START)
    assert torch.equal(d["motion_start_times"].cpu()[ids], s["t0"])
    close = lambda got, want, what: torch.testing.assert_close(got, want, atol=1e-5, rtol=0, msg=lambda m: f"{what}: {m}")
    close(d["root_states"].cpu()[ids], torch.cat([s["root_pos"], s["root_rot"], s["root_vel"], s["root_ang_vel"]], -1), "root_states")
    close(d["body_state"].cpu()[ids, :52], torch.cat([s["rb_pos"], s["rb_rot"], s["body_vel"], s["body_ang_vel"]], -1), "body_state")
    close(d["dof_pos"].cpu()[ids], s["dof_pos"], "dof_pos")
    close(d["dof_vel"].cpu()[ids], s["dof_vel"], "dof_vel")
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids] = False
    for k in ("root_states", "dof_pos", "body_state", "progress_buf", "contact_forces"):
        assert torch.equal(d[k].cpu()[keep], st[k][keep]), f"{k} of an env not reset"
    assert bool((d["body_state"].cpu()[ids, 52] == st["body_state"][ids, 52]).all())   # the other actor's body is not touched
    for k in ("progress_buf", "reset_buf", "terminate_buf"):
        assert int(d[k].cpu()[ids].abs().sum()) == 0, k
    assert float(d["contact_forces"].cpu()[ids].abs().sum()) == 0.0


def test_reset_matches_the_reference_fixture():
    """The device reset and _reset_task replaying the draws the reference's HumanoidSpeed reset methods recorded on a 52-body MotionLib
    (tests/golden/make_golden_smplx_speed.py): clips and start times bit-exact, the scattered state within 2e-5, task draws exact."""
    import os

    import numpy as np
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ztask_reset import ZTaskResetB200
    from tests.test_smplx_speed_cpu import reset_draws, reset_tables
    m = gen()
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smplx_speed.npz"))
    n = m.RESET_N
    ids, d = reset_draws(g, n)
    tb, floor = reset_tables(m)
    ml = MotionLibB200.from_tables(so.table_dict(tb), device=DEV)
    ml._sampling_batch_prob = torch.from_numpy(g["r_prob"]).to(DEV)
    r = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False)
    z = lambda *s, **k: torch.zeros(*s, device=DEV, **k)
    st = dict(root_states=z(n, 13), dof_pos=z(n, 153), dof_vel=z(n, 153), rigid_body_state=z(n, 53, 13),
              progress_buf=torch.ones(n, dtype=torch.int64, device=DEV), sampled_motion_ids=z(n, dtype=torch.int64), motion_start_times=z(n))
    ws = r.reset_envs(**st, env_ids=ids.to(DEV), motion_ids=d["motion_ids"].to(DEV), phase=d["phase"].to(DEV))
    # _reset_task as the fixture ran it: on the progress counters it found
    prog = torch.from_numpy(g["r_progress"]).to(DEV)
    tar, chg = torch.ones(n, device=DEV), z(n, dtype=torch.int64)
    r.reset_task(progress_buf=prog, change_steps=chg, tar_speed=tar, rand=d["task_u"].to(DEV), steps=d["steps"].to(DEV))
    torch.cuda.synchronize()
    T = lambda k: torch.from_numpy(g[k])[ids]
    assert torch.equal(ws["env_list"][:int(ws["count"].item())].cpu(), ids)
    assert torch.equal(st["sampled_motion_ids"].cpu()[ids], T("r_motion_ids")) and torch.equal(st["motion_start_times"].cpu()[ids], T("r_start_times"))
    close = lambda a, k: torch.testing.assert_close(a.cpu()[ids], T(k), atol=2e-5, rtol=0, msg=lambda x: f"{k}: {x}")
    close(st["root_states"], "r_root_states")
    close(st["rigid_body_state"][:, :52], "r_body_state")
    close(st["dof_pos"], "r_dof_pos")
    close(st["dof_vel"], "r_dof_vel")
    assert torch.equal(tar.cpu()[ids], T("r_tar_speed")) and torch.equal(chg.cpu()[ids], T("r_change_steps"))
    assert int(st["progress_buf"].cpu()[ids].abs().sum()) == 0


def test_reset_rejects_what_it_does_not_serve(motion):
    from pulse_b200 import PulseError
    from pulse_b200.ztask_reset import ZTaskResetB200
    _, ml, floor = motion
    with pytest.raises(PulseError, match="speed"):
        ZTaskResetB200("strike", ml, floor.to(DEV), upright=False)
    with pytest.raises(PulseError, match="upright=False"):
        ZTaskResetB200("speed", ml, floor.to(DEV), upright=True)
    with pytest.raises(PulseError, match="SMPL-X"):
        ml.handle                                               # the SMPL entry points never see the SMPL-X handle
    from pulse_b200.humanoid_im import HumanoidImCompute
    with pytest.raises(PulseError, match="SMPL-X"):
        HumanoidImCompute(ml)
    r = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False)
    n = 8
    z = lambda *s, **k: torch.zeros(*s, device=DEV, **k)
    kw = dict(root_states=z(n, 13), dof_pos=z(n, 153), dof_vel=z(n, 153), rigid_body_state=z(n, 52, 13), progress_buf=z(n, dtype=torch.int64),
              sampled_motion_ids=z(n, dtype=torch.int64), motion_start_times=z(n), reset_buf=z(n, dtype=torch.int64))
    with pytest.raises(PulseError, match="AMP"):
        r.reset_envs(**kw, amp_obs_buf=z(n, 10, 195))
    with pytest.raises(PulseError, match="153"):
        r.reset_envs(**dict(kw, dof_pos=z(n, 69), dof_vel=z(n, 69)))
    with pytest.raises(PulseError, match="52"):
        r.reset_envs(**dict(kw, rigid_body_state=z(n, 24, 13)))


# ------------------------------------------------------------------------------------------------ the driver
def _driver(n, motion, T=4, use_graphs=True, seed=5):
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.vae import PulseVAE
    from pulse_b200.ztask_reset import ZTaskResetB200
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    from pulse_b200.ztasks import SmplxSpeedTaskB200
    _, ml, floor = motion
    g = torch.Generator().manual_seed(seed)
    task = SmplxSpeedTaskB200(n, DEV, contact_body_ids=(7, 3, 8, 4))
    task._tar_speed.copy_(5.0 * torch.rand(n, generator=g))
    task._speed_change_steps.copy_(torch.randint(0, 320, (n,), generator=g))
    body = torch.zeros(n, 53, 13)
    body[..., 0:3] = torch.randn(n, 53, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 53, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 53, 6, generator=g)
    contact = torch.zeros(n, 53, 3)
    body[::7, 40, 2], contact[::7, 40, 2] = 0.05, 5.0                  # a hand on the ground: falls at progress > 1
    dof_state = torch.randn(n, 153, 2, generator=g)
    sim = dict(body_state=body, root_all=torch.randn(n, 2, 13, generator=g), dof_state=dof_state, contact_forces=contact,
               progress_buf=torch.randint(2, 300, (n,), generator=g), sampled_motion_ids=torch.randint(0, CLIPS, (n,), generator=g),
               motion_start_times=torch.rand(n, generator=g), actor_ids=torch.arange(n, dtype=torch.int32) * 2)
    sim = {k: v.to(DEV) for k, v in sim.items()}
    sim["root_all"][:, 0] = sim["body_state"][:, 0]
    sim.update(root_states=sim["root_all"][:, 0], dof_pos=sim["dof_state"][:, :, 0], dof_vel=sim["dof_state"][:, :, 1])
    policy = PPOPolicy(obs_size=task.obs_size, num_actions=48, units=(2048, 1024, 512), act="silu", device=DEV, seed=0)
    vae = PulseVAE(self_obs_size=778, num_actions=153, latent=48, device=DEV, with_critic=False, seed=1)
    reset = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False)
    drv = ZTaskStepsB200(task, reset, policy, vae, sim, horizon=T, pd_offset=torch.randn(153, generator=g).to(DEV),
                         pd_scale=(0.5 + torch.rand(153, generator=g)).to(DEV), use_graphs=use_graphs, reset_seed=3)
    drv.first_observation()
    return drv


def _state(drv):
    out = {k: getattr(drv, k) for k in ("obses", "obs_carry", "actions", "mus", "neglogp", "values", "next_values", "rewards", "dones", "pd_tar",
                                        "reset_buf", "terminate_buf")}
    out.update({k: drv.sim[k] for k in ("body_state", "root_all", "dof_state", "contact_forces", "progress_buf", "sampled_motion_ids",
                                        "motion_start_times")})
    out.update(tar_speed=drv.task._tar_speed, change=drv.task._speed_change_steps, prev_root=drv.task._prev_root_pos)
    return out


@pytest.mark.parametrize("n", [1536, 8192])
def test_horizon_graph_equals_eager_then_train(n, motion):
    a, b = _driver(n, motion, use_graphs=True), _driver(n, motion, use_graphs=False)
    resets = 0
    for use in ("eager", "capture", "replay"):
        a.play_steps()
        b.play_steps()
        sa, sb = _state(a), _state(b)
        for k in sa:
            assert torch.equal(sa[k], sb[k]), f"{use}: {k} differs"
        resets += float(a.dones.sum())
    assert resets > 0 and bool(torch.isfinite(a.obses).all())
    assert isinstance(a._graphs[("horizon",)], torch.cuda.CUDAGraph)
    a.finish()
    stats = a.train_epoch(mini_epochs=2, minibatch=4096 if n * a.T % 4096 == 0 else n * a.T)
    assert bool(torch.isfinite(stats).all()) and bool(torch.isfinite(a.policy.logstd).all())


def test_latent_post_at_48(motion):
    from tests.fp64_ref import latent_post_ref, philox_pair_normals
    drv = _driver(1536, motion, T=2, use_graphs=False)
    pol, vae = drv.policy, drv.vae
    obs = drv.obses[:, 0]
    obs.copy_(drv.obs_carry)
    prior_head, dec_in = vae.z_prior(obs)
    before = int(pol.rng_offset.item())
    drv._act(0)
    torch.cuda.synchronize()
    nrm, ntol = philox_pair_normals(pol.rng_seed, 1536, 48, before)
    ref = latent_post_ref(drv.mus[:, 0], nrm.to(DEV), pol.logstd, prior_head[:, :48], drv.actions[:, 0], eps_tol=ntol.to(DEV))
    for name, got in (("actions", drv.actions[:, 0]), ("neglogp", drv.neglogp[:, 0])):
        val, tol = ref[name]
        assert bool(((got.double() - val.double()).abs() <= tol.double()).all()), name
    assert torch.equal(dec_in[:, :48], ref["z"])
