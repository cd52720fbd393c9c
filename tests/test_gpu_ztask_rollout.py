"""The latent-space tasks' rollout on the device (`pulse_b200.ztask_rollout.ZTaskStepsB200`) and its kernels `pulse_latent_post`,
`pulse_ztask_pre_physics`, `pulse_reach_rollout_step` / `pulse_ztask_rollout_step`.

Bars: the fused kernels against torch (1e-6 / 1e-5) and, bit for bit, against the launches they replace; the graph-captured,
stream-overlapped horizon against the sequential eager one bit for bit over eager, capture and replay; `finish` and `train_epoch`
against the same calls issued separately; a replayed iteration without host synchronisation; the decode against
`PulseVAE.compute_z_actions`.  Fixtures are seeded synthetic state; every case runs once."""
import ctypes as C

import pytest
import torch

from tests.helpers import exact_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIPS = 23
KINDS = ("reach", "speed", "strike")
UNITS = (2048, 1024, 512)


@pytest.fixture(scope="module")
def motion():
    from pulse_b200.motion_lib import MotionLibB200
    tb = exact_tables(CLIPS, seed=9, min_frames=4, spread=120)
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames",
                                                                 "dt", "length_starts")}, device=DEV)
    g = torch.Generator().manual_seed(2)
    floor = (-0.9 + 0.05 * torch.rand(tb.motion_aa.shape[0], generator=g)).to(DEV)
    return ml, floor


def _sim(kind, n, seed):
    """Isaac-Gym shaped simulator tensors (2 actors per env, 72 dofs x (pos, vel), 26 bodies).  Every 7th env lies below its
    termination height with a contact force, and the progress counters reach the episode length inside a horizon."""
    g = torch.Generator().manual_seed(seed)
    body = torch.zeros(n, 26, 13)
    body[..., 0:3] = torch.randn(n, 26, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 26, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 26, 6, generator=g)
    contact = torch.zeros(n, 26, 3)
    body[::7, 5, 2], contact[::7, 5, 2] = 0.05, 5.0
    root = torch.randn(n, 2, 13, generator=g)
    root[:, 0] = body[:, 0]
    root[:, 1, 3:7] = torch.nn.functional.normalize(root[:, 1, 3:7], dim=-1)
    sim = dict(body_state=body, root_all=root, dof_state=torch.randn(n, 72, 2, generator=g), contact_forces=contact,
               progress_buf=torch.randint(2, 300, (n,), generator=g), sampled_motion_ids=torch.randint(0, CLIPS, (n,), generator=g),
               motion_start_times=torch.rand(n, generator=g), actor_ids=torch.arange(n, dtype=torch.int32) * 2,
               tar_contact_forces=60.0 * torch.randn(n, 3, generator=g))
    sim = {k: v.to(DEV) for k, v in sim.items()}
    sim.update(root_states=sim["root_all"][:, 0], dof_pos=sim["dof_state"][:, :69, 0], dof_vel=sim["dof_state"][:, :69, 1])
    if kind == "strike":
        sim.update(target_states=sim["root_all"][:, 1], tar_actor_ids=sim["actor_ids"] + 1)
    return sim


def _driver(kind, n, motion, T=4, seed=5, use_graphs=True, units=UNITS):
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.reach import ReachTaskB200
    from pulse_b200.vae import PulseVAE
    from pulse_b200.ztask_reset import ZTaskResetB200
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    from pulse_b200.ztasks import SpeedTaskB200, StrikeTaskB200
    ml, floor = motion
    task = {"reach": ReachTaskB200, "speed": SpeedTaskB200, "strike": StrikeTaskB200}[kind](n, device=DEV)
    g = torch.Generator().manual_seed(seed + 1)
    if kind == "reach":
        task._tar_pos.copy_(torch.randn(n, 3, generator=g))
        task._tar_change_steps.copy_(torch.randint(0, 320, (n,), generator=g))
    elif kind == "speed":
        task._tar_speed.copy_(5.0 * torch.rand(n, generator=g))
        task._speed_change_steps.copy_(torch.randint(0, 320, (n,), generator=g))
    reset = ZTaskResetB200(kind, ml, floor)
    policy = PPOPolicy(obs_size=task.obs_size, num_actions=32, units=units, act="silu", device=DEV, seed=0)
    vae = PulseVAE(device=DEV, with_critic=False, seed=1)
    pd_off = torch.randn(69, generator=g).to(DEV)
    pd_scale = (0.5 + torch.rand(69, generator=g)).to(DEV)
    freeze = torch.zeros(69, dtype=torch.uint8)
    freeze[[9, 10, 11, 66, 67, 68]] = 1
    drv = ZTaskStepsB200(task, reset, policy, vae, _sim(kind, n, seed), horizon=T, pd_offset=pd_off, pd_scale=pd_scale, pd_freeze=freeze.to(DEV),
                         use_graphs=use_graphs, reset_seed=3)
    drv.first_observation()
    return drv


def _state(drv):
    s, task = drv.sim, drv.task
    out = {k: getattr(drv, k) for k in ("obses", "obs_carry", "actions", "mus", "neglogp", "values", "next_values", "rewards", "dones", "pd_tar",
                                        "reset_buf", "terminate_buf")}
    out.update({k: s[k] for k in ("body_state", "root_all", "dof_state", "contact_forces", "progress_buf", "sampled_motion_ids", "motion_start_times")})
    if drv.kind == "reach":
        out.update(tar_pos=task._tar_pos, change=task._tar_change_steps)
    elif drv.kind == "speed":
        out.update(tar_speed=task._tar_speed, change=task._speed_change_steps, prev_root=task._prev_root_pos)
    else:
        out.update(prev_root=task._prev_root_pos)
    return out


def _assert_same(a, b, what=""):
    sa, sb = _state(a), _state(b)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f"{what}: {k} differs"


# ------------------------------------------------------------------------------------------------ 1. pulse_latent_post
@pytest.mark.parametrize("philox", [False, True])
def test_latent_post(philox):
    from pulse_b200 import _lib
    lib = _lib.load()
    n, T, E = 1027, 3, 32
    g = torch.Generator().manual_seed(11)
    mus = torch.randn(n, T, E, generator=g).to(DEV)
    prior = torch.randn(n, 2 * E, generator=g).to(DEV)
    value = torch.randn(n, 1, generator=g).to(DEV) * 3
    eps = None if philox else torch.randn(n, E, generator=g).to(DEV)
    logstd = (-2.9 + 0.3 * torch.randn(E, generator=g)).to(DEV)
    mean, var = torch.tensor([0.7], dtype=torch.float64, device=DEV), torch.tensor([2.3], dtype=torch.float64, device=DEV)
    offset = torch.tensor([12345], dtype=torch.int64, device=DEV)
    t = 1
    outs = []
    for fused in (True, False):
        actions, neglogp, values = torch.zeros(n, T, E, device=DEV), torch.zeros(n, T, device=DEV), torch.zeros(T, n, 1, device=DEV)
        dec_in = torch.full((n, 448), 7.0, device=DEV, dtype=torch.bfloat16)
        m, a_, nl, v = mus[:, t], actions[:, t], neglogp[:, t], values[t]
        common = dict(mu=m.data_ptr(), ld_mu=m.stride(0), logstd=logstd.data_ptr(), seed=99, rng_offset=offset.data_ptr(), rng_step=t,
                      actions=a_.data_ptr(), ld_actions=a_.stride(0), neglogp=nl.data_ptr(), ld_neglogp=nl.stride(0), value=value.data_ptr(),
                      ld_value=value.stride(0), value_mean=mean.data_ptr(), value_var=var.data_ptr(), value_eps=1e-5, values_out=v.data_ptr(),
                      ld_values=v.stride(0))
        if eps is not None:
            common.update(eps=eps.data_ptr(), ld_eps=eps.stride(0))
        st = _lib.current_stream(DEV)
        if fused:
            a = _lib.LatentPostArgs(latent=E, prior_mu=prior.data_ptr(), ld_prior=prior.stride(0), z_bf16=dec_in.data_ptr(), ld_z=dec_in.stride(0), **common)
            _lib.check(lib.pulse_latent_post(C.byref(a), n, st), "pulse_latent_post")
        else:
            a = _lib.PolicyPostArgs(num_actions=E, **common)
            _lib.check(lib.pulse_policy_post(C.byref(a), n, st), "pulse_policy_post")
            _lib.check(lib.pulse_vae_reparam(prior.data_ptr(), prior.stride(0), a_.data_ptr(), a_.stride(0), n, E, _lib.Z_RESIDUAL, 0, 0.0, 0.0,
                                             dec_in.data_ptr(), dec_in.stride(0), None, 0, st), "pulse_vae_reparam")
        outs.append((actions, neglogp, values, dec_in))
    for x, y, name in zip(outs[0], outs[1], ("actions", "neglogp", "values", "decoder operand")):
        assert torch.equal(x, y), f"{name}: the fused launch differs from pulse_policy_post + pulse_vae_reparam"
    actions, neglogp, values, dec_in = outs[0]
    assert float(actions[:, [0, 2]].abs().max()) == 0 and float((dec_in[:, E:].float() - 7.0).abs().max()) == 0    # other slices untouched
    act = actions[:, t]
    assert torch.equal(dec_in[:, :E], (prior[:, :E] + act).to(torch.bfloat16))
    torch.testing.assert_close(values[t], value.clamp(-5, 5) * torch.sqrt(var.float() + 1e-5) + mean.float(), atol=1e-6, rtol=1e-6)
    sg = torch.exp(logstd)
    if philox:
        e = (act - mus[:, t]) / sg
        assert abs(float(e.mean())) < 0.02 and abs(float(e.std()) - 1.0) < 0.02
    else:
        torch.testing.assert_close(act, mus[:, t] + sg * eps, atol=1e-6, rtol=1e-6)
        ref = 0.5 * (((act - mus[:, t]) / sg) ** 2).sum(-1) + 0.5 * 1.8378770664093453 * E + logstd.sum()
        torch.testing.assert_close(neglogp[:, t], ref, atol=1e-5, rtol=1e-5)


# ------------------------------------------------------------------------------------------------ 2. pulse_ztask_pre_physics
@pytest.mark.parametrize("kind", KINDS)
def test_pre_physics_injected(kind, motion):
    from pulse_b200.vae import pd_targets
    n = 1027
    drv = _driver(kind, n, motion, units=(64,))
    task, s = drv.task, drv.sim
    g = torch.Generator().manual_seed(21)
    dec = torch.randn(n, 80, generator=g).to(DEV)[:, :69]
    rand = (torch.rand(n, 3, generator=g) if kind == "reach" else torch.rand(n, generator=g)).to(DEV)
    steps = torch.randint(100, 200, (n,), generator=g).to(DEV)
    before = {k: v.clone() for k, v in _state(drv).items()}
    if kind != "strike":
        due = s["progress_buf"] >= before["change"]
        assert 0 < int(due.sum()) < n
        ref = {"reach": "_tar_pos", "speed": "_tar_speed"}[kind]
        task.update_task(s["progress_buf"], rand, steps)                      # the existing method, same draws
        exp_tar, exp_change = getattr(task, ref).clone(), before["change"].clone()
        exp_change[due] = (s["progress_buf"] + steps)[due]
        getattr(task, ref).copy_(before["tar_pos" if kind == "reach" else "tar_speed"])
        (task._tar_change_steps if kind == "reach" else task._speed_change_steps).copy_(before["change"])
    drv._pre_physics(dec, 0, rand=None if kind == "strike" else rand, steps=None if kind == "strike" else steps)
    assert torch.equal(drv.pd_tar, pd_targets(dec, drv.pd[0], drv.pd[1], freeze=drv.pd_freeze))
    assert float(drv.pd_tar[:, [9, 10, 11, 66, 67, 68]].abs().max()) == 0
    if kind != "reach":
        assert torch.equal(task._prev_root_pos, s["root_states"][:, 0:3])
    if kind != "strike":
        tar = task._tar_pos if kind == "reach" else task._tar_speed
        change = task._tar_change_steps if kind == "reach" else task._speed_change_steps
        assert torch.equal(tar, exp_tar) and torch.equal(change, exp_change)
        assert torch.equal(tar[~due], before["tar_pos" if kind == "reach" else "tar_speed"][~due])   # non-due envs untouched
    for k in ("body_state", "root_all", "dof_state", "progress_buf", "obs_carry", "reset_buf"):
        assert torch.equal(_state(drv)[k], before[k]), k


@pytest.mark.parametrize("kind", ("reach", "speed"))
def test_pre_physics_philox(kind, motion):
    n = 4099
    drv = _driver(kind, n, motion, units=(64,))
    task, s = drv.task, drv.sim
    dec = torch.zeros(n, 69, device=DEV)
    tar = task._tar_pos if kind == "reach" else task._tar_speed
    change = task._tar_change_steps if kind == "reach" else task._speed_change_steps
    tar0, change0 = tar.clone(), change.clone()
    due = s["progress_buf"] >= change0
    runs = []
    for t in (0, 0, 1):
        tar.copy_(tar0)
        change.copy_(change0)
        drv._pre_physics(dec, t)
        runs.append((tar.clone(), change.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])       # the same (seed, offset) repeats
    assert not torch.equal(runs[0][0][due], runs[2][0][due])                                  # another offset differs
    new_tar, new_change = runs[0]
    assert torch.equal(new_tar[~due], tar0[~due]) and torch.equal(new_change[~due], change0[~due])
    d = (new_change - s["progress_buf"])[due]
    assert int(d.min()) >= 100 and int(d.max()) < 200
    if kind == "reach":
        x = new_tar[due]
        assert float(x[:, :2].abs().max()) <= 1.0 and float(x[:, 2].min()) >= 0.5 and float(x[:, 2].max()) <= 1.5
        assert abs(float(x[:, 0].mean())) < 0.1 and abs(float(x[:, 2].mean()) - 1.0) < 0.05
    else:
        x = new_tar[due]
        assert float(x.min()) >= 0.0 and float(x.max()) <= 5.0 and abs(float(x.mean()) - 2.5) < 0.25


# ------------------------------------------------------------------------------------------------ 3. rollout step entry points
@pytest.mark.parametrize("kind", KINDS)
def test_rollout_step_equals_advance_then_step(kind, motion):
    n, t = 1027, 1
    drv = _driver(kind, n, motion, units=(64,))
    task, s = drv.task, drv.sim
    kw = dict(contact_forces=s["contact_forces"])
    progress0 = s["progress_buf"].clone()
    s["progress_buf"].add_(1)                                                 # the plain path: advance, then the task's own step
    if kind == "strike":
        task.post_physics_step(s["body_state"], s["progress_buf"], s["target_states"], s["tar_contact_forces"], **kw)
    else:
        task.post_physics_step(s["body_state"], s["progress_buf"], **kw)
    s["progress_buf"].copy_(progress0)
    drv._env_step(t)
    assert torch.equal(s["progress_buf"], progress0 + 1)
    assert torch.equal(drv.obses[:, t + 1], task.obs_buf) and float(drv.obses[:, t].abs().max()) == 0
    assert torch.equal(drv.rewards[t], task.rew_buf)
    assert torch.equal(drv.reset_buf, task.reset_buf) and torch.equal(drv.terminate_buf, task._terminate_buf)
    assert torch.equal(drv.dones[t], task.reset_buf.float())
    assert 0 < int(drv.reset_buf.sum()) < n and int(drv.terminate_buf.sum()) > 0


# ------------------------------------------------------------------------------------------------ 4. horizon: graphs + streams vs eager
@pytest.mark.parametrize("n", [1027, 8192])
@pytest.mark.parametrize("kind", KINDS)
def test_horizon_graph_equals_sequential(kind, n, motion):
    T = 4
    a = _driver(kind, n, motion, T=T, use_graphs=True)
    b = _driver(kind, n, motion, T=T, use_graphs=False)
    _assert_same(a, b, "initial")
    seen = []

    def refresh(t, ws):                     # the list observation taken before _reset_task, through the task's own method
        cnt = int(ws["count"].item())
        ids = ws["env_list"][:cnt].clone()
        kw = {"target_states": b.sim["target_states"]} if kind == "strike" else {}
        b.task.observe_list(b.sim["body_state"], ws["env_list"], ws["count"], b.sim["progress_buf"], **kw)
        seen.append((t, ids, b.task.obs_buf[ids].clone()))

    resets = 0
    for use in ("eager", "capture", "replay"):
        seen.clear()
        b.refresh = refresh
        a.play_steps()
        b.play_steps()
        _assert_same(a, b, use)
        assert len(seen) == T
        for t, ids, rows in seen:
            resets += ids.numel()
            assert torch.equal(b.obses[ids, t], rows), f"{use}: observation of the envs reset at step {t}"
        a.finish()
        b.finish()
        assert torch.equal(a.adv, b.adv) and torch.equal(a.ret, b.ret)
    assert resets > 0
    assert isinstance(a._graphs[("horizon",)], torch.cuda.CUDAGraph)
    assert float(a.dones.sum()) > 0 and bool(torch.isfinite(a.obses).all())


# ------------------------------------------------------------------------------------------------ 5. hook mode
@pytest.mark.parametrize("kind", KINDS)
def test_hooks_run_as_graph_segments(kind, motion):
    n, T = 1027, 3
    a = _driver(kind, n, motion, T=T, use_graphs=True)
    b = _driver(kind, n, motion, T=T, use_graphs=False)

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
    for use in ("eager", "capture", "replay"):
        a.play_steps()
        b.play_steps()
        _assert_same(a, b, use)
    assert sum(int(c) for c in counts) > 0
    assert all(isinstance(a._graphs[(seg, t)], torch.cuda.CUDAGraph) for seg in ("reset", "act", "post") for t in range(T))


# ------------------------------------------------------------------------------------------------ 6-8. finish, train_epoch, no syncs
def test_finish_and_train_epoch(motion):
    from pulse_b200.rollout import discount_values
    n, T = 1024, 4
    a = _driver("reach", n, motion, T=T, use_graphs=True)
    b = _driver("reach", n, motion, T=T, use_graphs=False)
    for _ in range(3):
        for d in (a, b):
            d.play_steps()
        # finish against the pieces computed separately
        pol = b.policy
        adv, ret = discount_values(b.dones, b.values, b.rewards.unsqueeze(-1), b.next_values, gamma=0.99, tau=0.95, normalize_advantage=True)
        pol.value_rms.update(b.values.view(-1, 1))
        ret_n = pol.value_rms.normalize_values(ret.view(-1, 1)).view(-1)
        pol.value_rms.update(ret.view(-1, 1))
        a.finish()
        assert torch.equal(a.adv, adv) and torch.equal(a.ret, ret_n)
        for name in ("running_mean", "running_var", "count"):      # fp64 moments summed with atomics: equal up to the order of the sum
            x, y = getattr(a.policy.value_rms, name), getattr(pol.value_rms, name)
            torch.testing.assert_close(x, y, rtol=1e-12, atol=0)
            y.copy_(x)
        pol.value_rms._refresh()
        b.adv.copy_(adv)
        b.ret.copy_(ret_n)
        # train_epoch against the same train_minibatch calls issued eagerly
        stats = a.train_epoch(mini_epochs=2, minibatch=1024).clone()
        rows, mb = n * T, 1024
        pol.reset_stats()
        for _k in range(2):
            for i in range(rows // mb):
                r0, r1 = i * mb, (i + 1) * mb
                pol.train_minibatch(b.obses.view(rows, -1)[r0:r1], b.actions.view(rows, -1)[r0:r1], b.neglogp.view(rows)[r0:r1], b.adv[r0:r1],
                                    b.ret[r0:r1], old_mu=b.mus.view(rows, -1)[r0:r1])
        torch.testing.assert_close(stats, pol.stats, rtol=1e-12, atol=1e-9)        # fp64 loss sums formed with atomics: last bits
        assert torch.equal(a.policy.flat.params, pol.flat.params), (a.policy.flat.params - pol.flat.params).abs().max()
        torch.testing.assert_close(a.policy.obs_rms.running_mean, pol.obs_rms.running_mean, rtol=1e-12, atol=1e-15)
    assert float(stats.abs().sum()) > 0
    with pytest.raises(Exception):
        a.train_epoch(minibatch=1000)
    # a replayed iteration makes no host synchronisation
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a.play_steps()
        a.finish()
        a.train_epoch(mini_epochs=2, minibatch=1024)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 9. K20 end to end
@pytest.mark.parametrize("kind", ("reach", "strike"))
def test_decode_matches_compute_z_actions(kind, motion):
    """One step: the decoder output that feeds pd_tar equals PulseVAE.compute_z_actions on the same observation rows and latent actions.
    Both run the same bf16 GEMM chain on identical operands (latent_post is bit-equal to the reparameterisation launch), so: exact."""
    from pulse_b200.vae import pd_targets
    n = 1027
    drv = _driver(kind, n, motion, T=1, use_graphs=False)
    drv.play_steps()
    dec = drv.z_actions.clone()
    ref = drv.vae.compute_z_actions(drv.obses[:, 0], drv.actions[:, 0])
    assert torch.equal(dec, ref)
    assert torch.equal(drv.pd_tar, pd_targets(ref, drv.pd[0], drv.pd[1], freeze=drv.pd_freeze))
    assert float(dec.abs().max()) > 0
