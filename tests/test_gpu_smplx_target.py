"""The PULSE-X reach and strike tasks on the device (52-body SMPL-X humanoid, HumanoidReachZ / HumanoidStrikeZ with
robot=smplx_humanoid): `pulse_smplx_target_step`, its list observation and rollout step against the oracle restatement pinned by the
reference fixture (observation and reward within 1e-5, reset and terminate bit-exact; the three kernels' rows agree to the last bit
of a few self-observation columns, as the SMPL-X speed step's do) at 1, 300, 2051 and 16384 envs; the reset
`pulse_reset_smplx_target` against the oracle and replaying the reference's recorded draws, with the AMP back-fill; the driver's
graph-captured horizon bit for bit against the eager one with resets inside it, without synchronisation, then `train_epoch`; and the
driver with the discriminator."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import smplx_speed_oracle as so
from tests import smplx_target_oracle as to
from tests import ztask_reset_oracle as zo
from tests.test_gpu_smplx_amp import _check_backfill, _model, _reset_state
from tests.test_gpu_smplx_speed import motion  # noqa: F401  (module fixture)
from tests.test_smplx_target_cpu import FIXTURE, gen, reset_draws

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIPS = 17
FEET = (7, 3, 8, 4)


def _task(kind, n, z, contacts, sm, reach_id=36, strike_ids=(35, 36, 45)):
    from pulse_b200.ztasks import SmplxReachTaskB200, SmplxStrikeTaskB200
    if kind == "reach":
        task = SmplxReachTaskB200(n, DEV, reach_body_id=reach_id, contact_body_ids=contacts, max_episode_length=sm.MAX_LEN)
        task._tar_pos.copy_(z["tar_pos"].to(DEV))
    else:
        task = SmplxStrikeTaskB200(n, DEV, strike_body_ids=strike_ids, contact_body_ids=contacts, max_episode_length=sm.MAX_LEN, dt=sm.DT)
        task._prev_root_pos.copy_(z["prev_root_pos"].to(DEV))
    return task


def _views(z, extra=1):
    """Isaac-Gym shaped views: `extra` bodies after the humanoid's 52 (body 52 the target's), the target's root state inside an
    [N, 2, 13] actor tensor and its contact force as body 52 of the contact tensor."""
    n = z["body_state"].shape[0]
    rb = torch.full((n, so.BODIES + extra, 13), 5.0, device=DEV)
    rb[:, :so.BODIES] = z["body_state"].to(DEV)
    cf = torch.zeros(n, so.BODIES + extra, 3, device=DEV)
    cf[:, :so.BODIES] = z["contact_forces"].to(DEV)
    cf[:, so.BODIES] = z["tar_contact_forces"].to(DEV)
    roots = torch.zeros(n, 2, 13, device=DEV)
    roots[:, 1] = z["target_states"].to(DEV)
    return rb, cf, roots[:, 1], cf[:, so.BODIES]


def _check(kind, z, contacts, sm, obs, rew, reset, term, rows=None, **ids):
    want_obs, want_rew, want_rs, want_tm = to.step(z, kind, contacts, sm.MAX_LEN, sm.DT, **ids)
    if rows is not None:
        want_obs = want_obs[rows]
    torch.testing.assert_close(obs.cpu(), want_obs, atol=1e-5, rtol=0)
    if rew is not None:
        torch.testing.assert_close(rew.cpu(), want_rew, atol=1e-5, rtol=0)
        assert torch.equal(reset.cpu(), want_rs) and torch.equal(term.cpu(), want_tm)


@pytest.mark.parametrize("contact_set", ["feet", "feet_and_bodies_above_31"])
@pytest.mark.parametrize("n", [1, 300, 2051, 16384])
@pytest.mark.parametrize("kind", ["reach", "strike"])
def test_step_list_and_rollout_rows(kind, n, contact_set):
    from pulse_b200 import _lib
    m = gen()
    sm = m.speed_gen()
    contacts = sm.CONTACT_IDS if contact_set == "feet" else sm.CONTACT_IDS_HI
    z = m.inputs(n, seed=n)
    rb, cf, ts, tcf = _views(z)
    prog = z["progress_buf"].to(DEV)
    for body in (m.REACH_IDS if kind == "reach" else (None,)):
        ids = dict(reach_id=body) if kind == "reach" else dict(strike_ids=m.STRIKE_IDS)
        task = _task(kind, n, z, contacts, sm, **ids)
        extra = dict(target_states=ts) if kind == "strike" else {}
        if kind == "strike":
            task.post_physics_step(rb, prog, ts, tcf, cf)
        else:
            task.post_physics_step(rb, prog, cf)
        torch.cuda.synchronize()
        _check(kind, z, contacts, sm, task.obs_buf, task.rew_buf, task.reset_buf, task._terminate_buf, **ids)
        # the list observation writes the listed rows (within 1e-5 of the oracle, as the step) and nothing else
        lst = torch.arange(0, n, 3, device=DEV)
        count = torch.tensor([lst.numel()], dtype=torch.int32, device=DEV)
        task.obs_buf.fill_(-7.0)
        task.observe_list(rb, lst, count, prog, contact_forces=cf, **extra)
        torch.cuda.synchronize()
        _check(kind, z, contacts, sm, task.obs_buf[lst], None, None, None, rows=lst.cpu(), **ids)
        keep = torch.ones(n, dtype=torch.bool, device=DEV)
        keep[lst] = False
        assert bool((task.obs_buf[keep] == -7.0).all())
        # the rollout step: progress += 1 inside the kernel, then the step (the oracle's rows, the step's reset and terminate words),
        # then dones = float(reset)
        reset0, term0 = task.reset_buf.clone(), task._terminate_buf.clone()
        p0 = (z["progress_buf"] - 1).to(DEV)
        dones = torch.full((n,), -1.0, device=DEV)
        a = task._args(rb, p0, cf)
        if kind == "strike":
            a.target_states, a.target_env_stride = ts.data_ptr(), ts.stride(0)
            a.tar_contact_forces, a.tar_contact_env_stride = tcf.data_ptr(), tcf.stride(0)
        task.obs_buf.zero_()
        _lib.check(task.lib.pulse_smplx_target_rollout_step(C.byref(a), dones.data_ptr(), n, _lib.current_stream(DEV)), "rollout")
        torch.cuda.synchronize()
        assert torch.equal(p0, prog)
        _check(kind, z, contacts, sm, task.obs_buf, task.rew_buf, task.reset_buf, task._terminate_buf, **ids)
        assert torch.equal(task.reset_buf, reset0) and torch.equal(task._terminate_buf, term0)
        assert torch.equal(dones, task.reset_buf.float())
    if kind == "strike" and n >= 300:
        pushed, strike_only = torch.arange(4, n, 13), torch.arange(6, n, 13)
        pushed, strike_only = pushed[z["progress_buf"][pushed] > 1], strike_only[z["progress_buf"][strike_only] > 1]
        assert bool((task._terminate_buf.cpu()[pushed] == 1).all()) and bool((task._terminate_buf.cpu()[strike_only] == 0).all())


# ------------------------------------------------------------------------------------------------ the reset
def _reset(kind, ml, floor, **kw):
    from pulse_b200.ztask_reset import SmplxTargetResetB200
    return SmplxTargetResetB200(kind, ml, floor.to(DEV), upright=False, **kw)


@pytest.mark.parametrize("state_init", ["Random", "Start"])
@pytest.mark.parametrize("kind", ["reach", "strike"])
def test_reset_matches_oracle(motion, kind, state_init):
    tb, ml, floor = motion
    n = 2051
    g = torch.Generator().manual_seed(8)
    st = _reset_state(n, 12)
    st["target_states"] = torch.randn(n, 2, 13, generator=g).to(DEV)[:, 1]
    before = {k: v.clone() for k, v in st.items()}
    motion_u, phase, strike_u = torch.rand(n, generator=g), torch.rand(n, generator=g), torch.rand(n, 4, generator=g)
    r = _reset(kind, ml, floor, state_init=state_init)
    kw = dict(strike_u=strike_u.to(DEV), target_states=st["target_states"]) if kind == "strike" else {}
    ws = r.reset_envs(**{k: v for k, v in st.items() if k != "target_states"}, motion_u=motion_u.to(DEV), phase=phase.to(DEV), **kw)
    torch.cuda.synchronize()
    ids = torch.nonzero(before["reset_buf"].cpu()).flatten()
    cnt = int(ws["count"].item())
    assert cnt == ids.numel() > 0 and torch.equal(ws["env_list"][:cnt].cpu(), ids)
    cdf = torch.cumsum(ml._sampling_batch_prob.cpu(), 0)
    clips = torch.searchsorted(cdf, torch.minimum(motion_u * cdf[-1], torch.nextafter(cdf[-1], torch.tensor(0.0))), right=True)
    assert torch.equal(st["sampled_motion_ids"].cpu()[ids], clips[ids])
    s = zo.sample_ref_state(tb, clips[ids], phase[ids], floor, zo.ROOT_XY_ZERO, False, zo.RANDOM if state_init == "Random" else zo.START)
    assert torch.equal(st["motion_start_times"].cpu()[ids], s["t0"])
    close = lambda got, want, what: torch.testing.assert_close(got, want, atol=1e-5, rtol=0, msg=lambda x: f"{what}: {x}")
    close(st["root_states"].cpu()[ids], torch.cat([s["root_pos"], s["root_rot"], s["root_vel"], s["root_ang_vel"]], -1), "root_states")
    close(st["rigid_body_state"].cpu()[ids, :52], torch.cat([s["rb_pos"], s["rb_rot"], s["body_vel"], s["body_ang_vel"]], -1), "body_state")
    close(st["dof_pos"].cpu()[ids], s["dof_pos"], "dof_pos")
    close(st["dof_vel"].cpu()[ids], s["dof_vel"], "dof_vel")
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids] = False
    if kind == "strike":
        close(st["target_states"].cpu()[ids], zo.reset_target(s["root_pos"][:, :2], strike_u[ids], **zo.STRIKE), "target_states")
    for k in ("root_states", "dof_pos", "rigid_body_state", "progress_buf", "contact_forces", "target_states"):
        assert torch.equal(st[k].cpu()[keep], before[k].cpu()[keep]), f"{k} of an env not reset"
    for k in ("progress_buf", "reset_buf", "terminate_buf"):
        assert int(st[k].cpu()[ids].abs().sum()) == 0, k


@pytest.mark.parametrize("kind", ["reach", "strike"])
def test_reset_replays_the_reference_fixture(kind):
    """The draws the reference's HumanoidReach / HumanoidStrike reset recorded on a 52-body MotionLib, replayed with the AMP buffer:
    clips and start times bit-exact, the state, targets and AMP history within 2e-5, reach's task draws exact."""
    from pulse_b200.motion_lib import MotionLibB200
    from tests.test_smplx_speed_cpu import reset_tables
    m = gen()
    sm = m.speed_gen()
    g = np.load(FIXTURE)
    n = sm.RESET_N
    ids, d = reset_draws(g, kind, n)
    tb, floor = reset_tables(sm)
    ml = MotionLibB200.from_tables(so.table_dict(tb), device=DEV)
    ml._sampling_batch_prob = torch.tensor(sm.PROB, device=DEV)
    r = _reset(kind, ml, floor)
    z = lambda *s, **k: torch.zeros(*s, device=DEV, **k)
    st = dict(root_states=z(n, 13), dof_pos=z(n, 153), dof_vel=z(n, 153), rigid_body_state=z(n, 53, 13),
              progress_buf=torch.ones(n, dtype=torch.int64, device=DEV), sampled_motion_ids=z(n, dtype=torch.int64), motion_start_times=z(n))
    buf, tgt = z(n, m.AMP_STEPS, m.AMP_WIDTH), z(n, 13)
    kw = dict(target_states=tgt, strike_u=d["strike_u"].to(DEV)) if kind == "strike" else {}
    r.reset_envs(**st, env_ids=ids.to(DEV), motion_ids=d["motion_ids"].to(DEV), phase=d["phase"].to(DEV), amp_obs_buf=buf, **kw)
    p = f"{kind}_r_"
    T = lambda k: torch.from_numpy(g[p + k])
    close = lambda a, k, want=None: torch.testing.assert_close(a, T(k)[ids] if want is None else want, atol=2e-5, rtol=0, msg=lambda x: f"{k}: {x}")
    if kind == "reach":
        prog, tar, chg = torch.from_numpy(g[p + "progress"]).to(DEV), z(n, 3), z(n, dtype=torch.int64)
        r.reset_task(progress_buf=prog, change_steps=chg, tar_pos=tar, rand=d["task_u"].to(DEV), steps=d["steps"].to(DEV))
        torch.cuda.synchronize()
        close(tar.cpu()[ids], "tar_pos")
        assert torch.equal(chg.cpu()[ids], T("change_steps")[ids])
    torch.cuda.synchronize()
    assert torch.equal(st["sampled_motion_ids"].cpu()[ids], T("motion_ids")[ids]) and torch.equal(st["motion_start_times"].cpu()[ids], T("start_times")[ids])
    close(st["root_states"].cpu()[ids], "root_states")
    close(st["rigid_body_state"].cpu()[ids, :52], "body_state", T("body_state"))
    close(st["dof_pos"].cpu()[ids], "dof_pos", T("dof_pos"))
    close(st["dof_vel"].cpu()[ids], "dof_vel", T("dof_vel"))
    if kind == "strike":
        close(tgt.cpu()[ids], "target_states")
    k = T("amp_obs").shape[0]
    torch.testing.assert_close(buf.cpu()[ids[:k]], T("amp_obs"), atol=2e-5, rtol=0)


@pytest.mark.parametrize("width", [465, 466])
@pytest.mark.parametrize("kind", ["reach", "strike"])
def test_reset_backfill_leaves_the_state_bit_identical(motion, kind, width):
    tb, ml, floor = motion
    n = 2051
    r = _reset(kind, ml, floor, amp_root_height_obs=width == 466)
    plain, st = _reset_state(n, 13), _reset_state(n, 13)
    tp, tt = torch.zeros(n, 13, device=DEV), torch.zeros(n, 13, device=DEV)
    buf = torch.full((n, 10, width), 7.0, device=DEV)
    fresh = torch.zeros(n, dtype=torch.int32, device=DEV)
    ws0 = r.reset_envs(**plain, seed=4, offset=2, **(dict(target_states=tp) if kind == "strike" else {}))
    cnt0, list0 = int(ws0["count"].item()), ws0["env_list"].clone()
    ws = r.reset_envs(**st, amp_obs_buf=buf, amp_fresh=fresh, seed=4, offset=2, **(dict(target_states=tt) if kind == "strike" else {}))
    torch.cuda.synchronize()
    assert int(ws["count"].item()) == cnt0 > 0 and torch.equal(ws["env_list"][:cnt0], list0[:cnt0])
    for k in plain:
        assert torch.equal(plain[k], st[k]), f"{k}: the AMP buffer changed the reset's state outputs"
    assert torch.equal(tp, tt)
    ids = list0[:cnt0]
    assert bool((st["root_states"][ids, 0:2] == 0).all())
    _check_backfill(tb, st, ids, buf, width)


def test_reset_refusals(motion):
    from pulse_b200 import PulseError
    from types import SimpleNamespace as NS

    from pulse_b200.ztask_reset import SmplxTargetResetB200, ZTaskResetB200
    _, ml, floor = motion
    with pytest.raises(PulseError, match="speed"):
        ZTaskResetB200("reach", ml, floor.to(DEV), upright=False)           # ZTaskResetB200 keeps serving SMPL-X speed only
    with pytest.raises(PulseError, match="reach and strike"):
        SmplxTargetResetB200("speed", ml, floor.to(DEV), upright=False)
    with pytest.raises(PulseError, match="upright=False"):
        SmplxTargetResetB200("strike", ml, floor.to(DEV), upright=True)
    with pytest.raises(PulseError, match="52-body"):
        SmplxTargetResetB200("reach", NS(smplx=False), floor.to(DEV), upright=False)


# ------------------------------------------------------------------------------------------------ the driver
def _driver(kind, n, motion, T=4, use_graphs=True, seed=5, amp_width=None):
    from pulse_b200.amp_buffers import AmpBuffersB200
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.vae import PulseVAE
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    from pulse_b200.ztasks import SmplxReachTaskB200, SmplxStrikeTaskB200
    _, ml, floor = motion
    g = torch.Generator().manual_seed(seed)
    if kind == "reach":
        task = SmplxReachTaskB200(n, DEV, reach_body_id=36, contact_body_ids=FEET)
        task._tar_pos.copy_(torch.randn(n, 3, generator=g))
        task._tar_change_steps.copy_(torch.randint(0, 320, (n,), generator=g))
    else:
        task = SmplxStrikeTaskB200(n, DEV, strike_body_ids=(35, 36, 45), contact_body_ids=FEET)
    body = torch.zeros(n, 53, 13)
    body[..., 0:3] = torch.randn(n, 53, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 53, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 53, 6, generator=g)
    contact = torch.zeros(n, 53, 3)
    body[::7, 40, 2], contact[::7, 40, 2] = 0.05, 5.0                  # a hand on the ground: falls at progress > 1
    contact[3::7, 20, 0], contact[3::7, 52, 0] = 70.0, 80.0            # strike: the target pushed while body 20 presses
    dof_state = torch.randn(n, 153, 2, generator=g)
    sim = dict(body_state=body, root_all=torch.randn(n, 2, 13, generator=g), dof_state=dof_state, contact_forces=contact,
               progress_buf=torch.randint(2, 300, (n,), generator=g), sampled_motion_ids=torch.randint(0, CLIPS, (n,), generator=g),
               motion_start_times=torch.rand(n, generator=g), actor_ids=torch.arange(n, dtype=torch.int32) * 2)
    sim = {k: v.to(DEV) for k, v in sim.items()}
    sim["root_all"][:, 0] = sim["body_state"][:, 0]
    sim.update(root_states=sim["root_all"][:, 0], dof_pos=sim["dof_state"][:, :, 0], dof_vel=sim["dof_state"][:, :, 1])
    if kind == "strike":
        sim.update(target_states=sim["root_all"][:, 1], tar_contact_forces=sim["contact_forces"][:, 52],
                   tar_actor_ids=torch.arange(n, dtype=torch.int32, device=DEV) * 2 + 1)
    disc = dict(with_disc=True, amp_obs_size=10 * amp_width, disc_units=(256, 128)) if amp_width else {}
    units = (256, 128) if amp_width else (2048, 1024, 512)
    policy = PPOPolicy(obs_size=task.obs_size, num_actions=48, units=units, act="silu", device=DEV, seed=0, **disc)
    vae = PulseVAE(self_obs_size=778, num_actions=153, latent=48, device=DEV, with_critic=False, seed=1)
    reset = _reset(kind, ml, floor, amp_root_height_obs=amp_width == 466)
    amp = None
    if amp_width:
        amp = AmpBuffersB200(ml, num_steps=10, amp_width=amp_width, upright=False, demo_buffer_size=160, replay_buffer_size=120, batch_size=64,
                             keep_prob=0.5, minibatch_size=16, seed=2)
    drv = ZTaskStepsB200(task, reset, policy, vae, sim, horizon=T, pd_offset=torch.randn(153, generator=g).to(DEV),
                         pd_scale=(0.5 + torch.rand(153, generator=g)).to(DEV), use_graphs=use_graphs, reset_seed=3, amp=amp)
    drv.first_observation()
    return drv


def _state(drv):
    out = {k: getattr(drv, k) for k in ("obses", "obs_carry", "actions", "mus", "neglogp", "values", "next_values", "rewards", "dones", "pd_tar",
                                        "reset_buf", "terminate_buf")}
    out.update({k: drv.sim[k] for k in ("body_state", "root_all", "dof_state", "contact_forces", "progress_buf", "sampled_motion_ids",
                                        "motion_start_times")})
    if drv.kind == "reach":
        out.update(tar=drv.task._tar_pos, change=drv.task._tar_change_steps)
    else:
        out.update(prev_root=drv.task._prev_root_pos)
    return out


@pytest.mark.parametrize("n", [1536, 8192])
@pytest.mark.parametrize("kind", ["reach", "strike"])
def test_horizon_graph_equals_eager_then_train(kind, n, motion):
    a, b = _driver(kind, n, motion, use_graphs=True), _driver(kind, n, motion, use_graphs=False)
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
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a.play_steps()                                                   # a replay makes no synchronisation
    finally:
        torch.cuda.set_sync_debug_mode("default")
    a.finish()
    stats = a.train_epoch(mini_epochs=2, minibatch=4096 if n * a.T % 4096 == 0 else n * a.T)
    assert bool(torch.isfinite(stats).all()) and bool(torch.isfinite(a.policy.logstd).all())


N, T, MB = 24, 4, 32


@pytest.mark.parametrize("kind", ["reach", "strike"])
def test_driver_with_discriminator(kind, motion):
    """AmpBuffersB200 at 465 floats and a discriminator of 4650 inputs, unchanged: the horizon's AMP rows equal the eager composition
    (row kernel over the state the step saw, history from the previous row or the reset's back-fill), graph equals eager, and
    train_epoch equals train_minibatch called by hand."""
    from tests import smplx_amp_fp64 as xf
    d = _driver(kind, N, motion, T=T, use_graphs=False, amp_width=465)
    assert d.policy.disc is not None and d.amp.amp_width == 465
    W, S = d.amp.amp_width, d.amp.num_steps
    snaps = {}

    def refresh(t, ws):
        s = d.sim
        snaps[t] = (s["body_state"][:, :52].clone(), s["dof_pos"].clone(), s["dof_vel"].clone(), d.amp_init.clone(), d.amp_fresh.clone() != 0)

    d.refresh = refresh
    H = d.amp_obs[:, T - 1].view(N, S, W).clone()
    d.play_steps()
    for t in range(T):
        body, dp, dv, init, fresh = snaps[t]
        got = d.amp_obs[:, t].view(N, S, W)
        xf.check_amp(None, f"{kind} step {t} current row", got[:, 0], xf.state_amp_ref(body, dp, dv))
        hist = torch.where(fresh[:, None, None], init[:, :S - 1], H[:, :S - 1])
        assert torch.equal(got[:, 1:], hist), f"step {t}: history rows"
        H = torch.cat([got[:, :1], hist], 1)
    # graph against eager
    a, b = _driver(kind, N, motion, T=T, use_graphs=True, amp_width=465), _driver(kind, N, motion, T=T, use_graphs=False, amp_width=465)
    for it in range(3):
        for x in (a, b):
            x.play_steps()
            x.finish()
            x.train_epoch(mini_epochs=2, minibatch=MB)
        for k in ("amp_obs", "amp_init", "amp_fresh", "obses", "rewards", "adv", "ret"):
            assert torch.equal(getattr(a, k), getattr(b, k)), f"iteration {it}: {k}"
        assert torch.equal(a.policy.flat.params, b.policy.flat.params), f"iteration {it}: parameters"
    # train_epoch against train_minibatch by hand
    a, b = _driver(kind, N, motion, T=T, use_graphs=False, amp_width=465), _driver(kind, N, motion, T=T, use_graphs=False, amp_width=465)
    rows, take = N * T, min(16, MB)
    for it in range(2):
        for x in (a, b):
            x.play_steps()
            x.finish()
        a.train_epoch(mini_epochs=2, minibatch=MB)
        amp, Wr = b.amp, b.amp.row_floats
        amp.update_demos()
        flat = b.amp_obs.view(rows, Wr)
        md, mr = _model(amp.demo), _model(amp.replay)
        demo = amp.demo.rows[torch.from_numpy(md.sample(rows)).to(DEV)]
        ri = mr.sample(rows)
        replay = flat.clone() if ri is None else amp.replay.rows[torch.from_numpy(ri).to(DEV)]
        for ring, mm in ((amp.demo, md), (amp.replay, mr)):
            ring.ctr[:5] = torch.from_numpy(mm.counters()).to(DEV)
        b.policy.reset_stats()
        for _ in range(2):
            for i in range(rows // MB):
                r0, r1 = i * MB, (i + 1) * MB
                b.policy.train_minibatch(b.obses.view(rows, -1)[r0:r1], b.actions.view(rows, -1)[r0:r1], b.neglogp.view(rows)[r0:r1],
                                         b.adv[r0:r1], b.ret[r0:r1], old_mu=b.mus.view(rows, -1)[r0:r1],
                                         amp=(flat[r0:r0 + take], replay[r0:r0 + take], demo[r0:r0 + take]))
        amp.store_replay(flat)
        assert torch.equal(a.policy.flat.params, b.policy.flat.params), f"iteration {it}: parameters"
        torch.testing.assert_close(a.policy.disc.stats, b.policy.disc.stats, rtol=1e-9, atol=0)
