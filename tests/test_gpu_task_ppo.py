"""The downstream tasks' PPO baseline on the device: reach, speed and strike trained from scratch with a dof-space policy
(HumanoidReach / HumanoidSpeed / HumanoidStrike under learning=ppo), for SMPL (69 actions) and SMPL-X (153 actions).

Bars: `pulse_policy_post` at 129, 153 and 256 actions element-wise against the fp64 reference, with injected draws and with the
kernel's Philox draws regenerated on the host at the wide layout; `pulse_ppo_loss` at 153 actions against fp64 autograd (with and
without old_mu); the 153-wide actor head of the ppo.yaml network link by link (forward, dgrad, weight gradient); `ZTaskStepsB200` with
`vae=None` bit for bit between the single-graph horizon, the hook-segment schedule and the eager one with resets inside the horizon,
PD targets equal to the torch composition, finite statistics and moved parameters after `train_epoch`, also with the discriminator;
a 153-action `state_dict` round trip.  Run with -s to print the margin of every fp64 link."""
import ctypes as C

import pytest
import torch

from tests import smplx_speed_oracle as so
from tests.fp64_links import _snapshot, check_grads, check_mlp, check_ppo_loss
from tests.fp64_ref import Report, check, f64, philox_pair_normals, policy_post_ref
from tests.helpers import exact_tables
from tests.test_gpu_ztask_rollout import _sim as smpl_sim
from tests.test_task_ppo_cpu import policy_post_stride

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UNITS = (2048, 1024, 512)            # ppo.yaml
KINDS = ("reach", "speed", "strike")
DOFS = {"smpl": 69, "smplx": 153}
SMPLX_CLIPS = 17
FEET = (7, 3, 8, 4)


@pytest.fixture(scope="module")
def motions():
    from pulse_b200.motion_lib import MotionLibB200
    tb = exact_tables(23, seed=9, min_frames=4, spread=120)
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames",
                                                                 "dt", "length_starts")}, device=DEV)
    g = torch.Generator().manual_seed(2)
    floor = (-0.9 + 0.05 * torch.rand(tb.motion_aa.shape[0], generator=g)).to(DEV)
    tbx = so.tables(SMPLX_CLIPS, seed=5)
    mlx = MotionLibB200.from_tables(so.table_dict(tbx), device=DEV)
    g = torch.Generator().manual_seed(3)
    floorx = (-0.9 + 0.05 * torch.rand(tbx.gts.shape[0], generator=g)).to(DEV)
    return {"smpl": (ml, floor), "smplx": (mlx, floorx)}


def _smplx_sim(kind, n, g):
    body = torch.zeros(n, 53, 13)
    body[..., 0:3] = torch.randn(n, 53, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 53, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 53, 6, generator=g)
    contact = torch.zeros(n, 53, 3)
    body[::7, 40, 2], contact[::7, 40, 2] = 0.05, 5.0                  # a hand on the ground: falls at progress > 1
    contact[3::7, 20, 0], contact[3::7, 52, 0] = 70.0, 80.0            # strike: the target pushed while body 20 presses
    sim = dict(body_state=body, root_all=torch.randn(n, 2, 13, generator=g), dof_state=torch.randn(n, 153, 2, generator=g), contact_forces=contact,
               progress_buf=torch.randint(2, 300, (n,), generator=g), sampled_motion_ids=torch.randint(0, SMPLX_CLIPS, (n,), generator=g),
               motion_start_times=torch.rand(n, generator=g), actor_ids=torch.arange(n, dtype=torch.int32) * 2)
    sim = {k: v.to(DEV) for k, v in sim.items()}
    sim["root_all"][:, 0] = sim["body_state"][:, 0]
    sim.update(root_states=sim["root_all"][:, 0], dof_pos=sim["dof_state"][:, :, 0], dof_vel=sim["dof_state"][:, :, 1])
    if kind == "strike":
        sim.update(target_states=sim["root_all"][:, 1], tar_contact_forces=sim["contact_forces"][:, 52],
                   tar_actor_ids=torch.arange(n, dtype=torch.int32, device=DEV) * 2 + 1)
    return sim


def _driver(layout, kind, n, motions, T=4, use_graphs=True, seed=5, amp=False, units=UNITS):
    """ZTaskStepsB200(vae=None) with a PPOPolicy that acts in the layout's dofs; `amp`: with the discriminator and AmpBuffersB200
    (SMPL: 195-float rows, upright False; SMPL-X: 465-float rows), task and discriminator rewards mixed half and half."""
    from pulse_b200.amp_buffers import AmpBuffersB200
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.ztask_reset import SmplxTargetResetB200, ZTaskResetB200
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    from pulse_b200 import reach, ztasks
    ml, floor = motions[layout]
    g = torch.Generator().manual_seed(seed)
    D = DOFS[layout]
    width, upright = (195, False) if layout == "smpl" else (465, False)
    if layout == "smpl":
        task = {"reach": reach.ReachTaskB200, "speed": ztasks.SpeedTaskB200, "strike": ztasks.StrikeTaskB200}[kind](n, device=DEV)
        sim = smpl_sim(kind, n, seed)
        reset = ZTaskResetB200(kind, ml, floor, **(dict(upright=upright, amp_root_height_obs=False) if amp else {}))
    else:
        if kind == "reach":
            task = ztasks.SmplxReachTaskB200(n, DEV, reach_body_id=36, contact_body_ids=FEET)
        elif kind == "speed":
            task = ztasks.SmplxSpeedTaskB200(n, DEV, contact_body_ids=FEET)
        else:
            task = ztasks.SmplxStrikeTaskB200(n, DEV, strike_body_ids=(35, 36, 45), contact_body_ids=FEET)
        sim = _smplx_sim(kind, n, g)
        cls = ZTaskResetB200 if kind == "speed" else SmplxTargetResetB200
        reset = cls(kind, ml, floor, upright=False, amp_root_height_obs=False)
    if kind == "reach":
        task._tar_pos.copy_(torch.randn(n, 3, generator=g))
        task._tar_change_steps.copy_(torch.randint(0, 320, (n,), generator=g))
    elif kind == "speed":
        task._tar_speed.copy_(5.0 * torch.rand(n, generator=g))
        task._speed_change_steps.copy_(torch.randint(0, 320, (n,), generator=g))
    disc = dict(with_disc=True, amp_obs_size=10 * width, disc_units=(256, 128)) if amp else {}
    policy = PPOPolicy(obs_size=task.obs_size, num_actions=D, units=units, act="silu", logstd=-2.9, device=DEV, seed=0, **disc)
    freeze = torch.zeros(D, dtype=torch.uint8)
    freeze[[9, 10, 11, D - 3, D - 2, D - 1]] = 1
    kw = {}
    if amp:
        kw = dict(amp=AmpBuffersB200(ml, num_steps=10, amp_width=width, upright=upright, demo_buffer_size=160, replay_buffer_size=120,
                                     batch_size=64, keep_prob=0.5, minibatch_size=16, seed=2), task_reward_w=0.5, disc_reward_w=0.5)
    drv = ZTaskStepsB200(task, reset, policy, None, sim, horizon=T, pd_offset=torch.randn(D, generator=g).to(DEV),
                         pd_scale=(0.5 + torch.rand(D, generator=g)).to(DEV), pd_freeze=freeze.to(DEV), use_graphs=use_graphs, reset_seed=3, **kw)
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
        if drv.kind == "speed":
            out.update(tar_speed=drv.task._tar_speed, change=drv.task._speed_change_steps)
    if drv.amp is not None:
        out.update(amp_obs=drv.amp_obs, amp_init=drv.amp_init, amp_fresh=drv.amp_fresh)
    return out


def _assert_same(drivers, what):
    ref = _state(drivers[0])
    for d in drivers[1:]:
        s = _state(d)
        for k in ref:
            assert torch.equal(ref[k], s[k]), f"{what}: {k} differs"


def _pd_composition(drv, t):
    off, scale = drv.pd
    v = off + scale * drv.actions[:, t]
    return torch.where(drv.pd_freeze.bool(), torch.zeros_like(v), v)


# ------------------------------------------------------------------------------------------------ 1. pulse_policy_post, wide
@pytest.mark.parametrize("noise", ["eps", "philox"])
@pytest.mark.parametrize("A", [129, 153, 256])
def test_policy_post_wide(A, noise):
    from pulse_b200 import _lib
    lib = _lib.load()
    M, T, t = 2051, 3, 1
    g = torch.Generator(device=DEV).manual_seed(A)
    mu_all = torch.randn(M, T, A, device=DEV, generator=g)
    mu = mu_all[:, t]                                                    # a strided experience slice
    logstd = -2.9 + 0.3 * torch.randn(A, device=DEV, generator=g)
    value = torch.randn(M, 1, device=DEV, generator=g) * 4
    mean = torch.full((1,), 0.7, dtype=torch.float64, device=DEV)
    var = torch.full((1,), 2.3, dtype=torch.float64, device=DEV)
    actions, nlp = torch.full((M, T, A), 7.0, device=DEV), torch.full((M, T), 7.0, device=DEV)
    values = torch.full((T, M, 1), 7.0, device=DEV)
    eps = torch.randn(M, A, device=DEV, generator=g) if noise == "eps" else None
    seed, off_dev, step = 0x243F6A8885A308D3, torch.tensor([1000], dtype=torch.int64, device=DEV), 5
    a = _lib.PolicyPostArgs(mu=mu.data_ptr(), ld_mu=mu.stride(0), logstd=logstd.data_ptr(), seed=seed, rng_offset=off_dev.data_ptr(), rng_step=step,
                            num_actions=A, actions=actions[:, t].data_ptr(), ld_actions=actions.stride(0), neglogp=nlp[:, t].data_ptr(),
                            ld_neglogp=nlp.stride(0), value=value.data_ptr(), ld_value=1, value_mean=mean.data_ptr(), value_var=var.data_ptr(),
                            value_eps=1e-5, values_out=values[t].data_ptr(), ld_values=1)
    if eps is not None:
        a.eps, a.ld_eps = eps.data_ptr(), eps.stride(0)
    _lib.check(lib.pulse_policy_post(C.byref(a), M, _lib.current_stream(DEV)), "pulse_policy_post")
    torch.cuda.synchronize()
    rep = Report(f"policy_post, A={A}, {noise}")
    try:
        if eps is None:
            n, nt = philox_pair_normals(seed, M, A, 1000 + step, stride=policy_post_stride(A))
            n, nt = n.to(DEV), nt.to(DEV)
            plain = policy_post_ref(mu, n, logstd)
            sg = torch.exp(f64(logstd))
            check(rep, "philox draws (a - mu) / sigma", (f64(actions[:, t]) - f64(mu)) / sg, n, nt + plain["actions"][1] / sg)
            ref = policy_post_ref(mu, n, logstd, eps_tol=nt, value=value, value_mean=mean, value_var=var, value_eps=1e-5)
        else:
            ref = policy_post_ref(mu, eps, logstd, value=value, value_mean=mean, value_var=var, value_eps=1e-5)
        check(rep, "actions", actions[:, t], *ref["actions"])
        check(rep, "neglogp", nlp[:, t], *ref["neglogp"])
        check(rep, "values (value_unnorm)", values[t].reshape(-1), ref["values"][0].reshape(-1), ref["values"][1].reshape(-1))
    finally:
        print("\n" + rep.text())
    keep = [i for i in range(T) if i != t]
    assert bool((actions[:, keep] == 7.0).all()) and bool((nlp[:, keep] == 7.0).all()) and bool((values[keep] == 7.0).all())


# ------------------------------------------------------------------------------------------------ 2-3. ppo_loss and the 153-wide head
def _wide_policy(seed):
    from pulse_b200.ppo import PPOPolicy
    pol = PPOPolicy(obs_size=781, num_actions=153, units=UNITS, act="silu", logstd=-2.9, device=DEV, seed=seed)
    head = pol.actor.layers[-1]
    with torch.no_grad():             # a few action heads past the soft bound so the bounds loss has active elements
        head.weight[:4, head.K] = torch.tensor([1.5, -1.5, 1.2, -1.2], device=DEV)
        head.weight[150:153, head.K] = torch.tensor([1.3, -1.3, 1.1], device=DEV)
        head.refresh()
    g = torch.Generator(device=DEV).manual_seed(seed + 100)
    pol.obs_rms.update(torch.randn(4096, 781, device=DEV, generator=g) * 1.3 + 0.1)
    return pol, g


def _ppo_inputs(pol, M, g):
    obs = torch.randn(M, 781, device=DEV, generator=g) * 1.5 + 0.2
    out = pol.act(obs, eps=torch.randn(M, 153, device=DEV, generator=g))
    actions, nlp, mus = out["actions"].clone().contiguous(), out["neglogpacs"].clone(), out["mus"].clone().contiguous()
    adv = torch.randn(M, device=DEV, generator=g)
    grp = torch.arange(M, device=DEV) % 4
    nlp = nlp + torch.where(grp == 1, 0.4, torch.where(grp == 2, -0.4, torch.where(grp == 3, 0.4, 0.0)))
    adv = torch.where(grp == 1, adv.abs() + 0.1, torch.where(grp >= 2, -(adv.abs() + 0.1), adv))
    ret = torch.randn(M, device=DEV, generator=g)
    return obs, actions, nlp, adv, ret, mus


@pytest.mark.parametrize("M", [4096, 2051])
def test_ppo_loss_and_actor_head_153_fp64(M):
    pol, g = _wide_policy(seed=M)
    obs, actions, old_nlp, adv, ret, mus = _ppo_inputs(pol, M, g)
    snap = _snapshot(pol.flat)
    rep = Report(f"PPO update, 153 actions, M={M}")
    try:
        pol.reset_stats()
        pol.train_minibatch(obs, actions, old_nlp, adv, ret, old_mu=mus, keep_grads=True)
        torch.cuda.synchronize()
        b = pol._buf(M, True)
        x = b["x2"][0]
        wa, ba = check_mlp(rep, "actor", pol.actor, snap, x, b["dmu"], M)
        wc, bc = check_mlp(rep, "critic", pol.critic, snap, x, b["dv"], M)
        check_ppo_loss(rep, pol, M, actions, old_nlp, adv, ret, mus)
        check_grads(rep, "actor", pol.actor, wa, ba)
        check_grads(rep, "critic", pol.critic, wc, bc)
        # without old_mu: the same gradients, the same statistics but the KL sum, which is 0
        from pulse_b200 import _lib
        mu, value = pol.actor._ws[(M, True)]["out"][:M], pol.critic._ws[(M, True)]["out"][:M]
        outs = []
        for old in (mus, None):
            dmu = torch.zeros(M, 160, device=DEV, dtype=torch.bfloat16)
            dv = torch.zeros(M, 8, device=DEV, dtype=torch.bfloat16)
            st = torch.zeros(6, dtype=torch.float64, device=DEV)
            a = _lib.PpoLossArgs(mu=mu.data_ptr(), ld_mu=mu.stride(0), value=value.data_ptr(), ld_value=value.stride(0), actions=actions.data_ptr(),
                                 old_neglogp=old_nlp.data_ptr(), advantages=adv.data_ptr(), returns=ret.data_ptr(),
                                 old_mu=old.data_ptr() if old is not None else None, logstd=pol.logstd.data_ptr(), num_actions=153,
                                 e_clip=pol.e_clip, critic_coef=pol.critic_coef, bounds_coef=pol.bounds_coef, dmu=dmu.data_ptr(), ld_dmu=160,
                                 dvalue=dv.data_ptr(), ld_dv=8, stats=st.data_ptr())
            _lib.check(pol.lib.pulse_ppo_loss(C.byref(a), M, _lib.current_stream(DEV)), "pulse_ppo_loss")
            outs.append((dmu, dv, st))
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        assert torch.equal(outs[0][0][:, :153], b["dmu"][:M, :153])
        assert float(outs[1][2][3]) == 0.0 and float(outs[0][2][3]) != 0.0     # the KL term at equal means is log(1 + 1e-5) - 0.5 + ...
        keep = [0, 1, 2, 4, 5]
        torch.testing.assert_close(outs[0][2][keep], outs[1][2][keep], rtol=1e-12, atol=1e-9)   # fp64 atomics: summation order
    finally:
        print("\n" + rep.text())


def test_state_dict_round_trip_153():
    from pulse_b200.ppo import PPOPolicy
    pol, g = _wide_policy(seed=11)
    with torch.no_grad():
        pol.logstd.add_(0.01 * torch.randn(153, device=DEV, generator=g))
    pol.value_rms.update(torch.randn(512, 1, device=DEV, generator=g))
    sd = pol.state_dict()
    assert tuple(sd["a2c_network.mu.weight"].shape) == (153, 512) and tuple(sd["a2c_network.mu.bias"].shape) == (153,)
    assert tuple(sd["a2c_network.sigma"].shape) == (153,)
    assert tuple(sd["a2c_network.actor_mlp.0.weight"].shape) == (2048, 781) and tuple(sd["a2c_network.value.weight"].shape) == (1, 512)
    fresh = PPOPolicy(obs_size=781, num_actions=153, units=UNITS, act="silu", logstd=-1.0, device=DEV, seed=99)
    fresh.load_state_dict(sd)
    obs = torch.randn(2051, 781, device=DEV, generator=g)
    outs = []
    for p in (pol, fresh):
        mus = torch.zeros(2051, 4, 153, device=DEV)[:, 2]
        v = p.heads_into(obs, mus=mus).clone()
        outs.append((mus.clone(), v))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(pol.logstd, fresh.logstd)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, sd[k]), k


# ------------------------------------------------------------------------------------------------ 4. the driver
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", ["smpl", "smplx"])
def test_driver_graph_segments_eager_then_train(layout, kind, motions):
    """2051 envs (not a multiple of the 128-thread blocks), T = 4: the single graph, the hook segments (a refresh hook that does
    nothing) and the eager horizon agree bit for bit over eager, capture and replay, with resets inside every horizon."""
    n, T = 2051, 4
    a = _driver(layout, kind, n, motions, T=T, use_graphs=True)
    s = _driver(layout, kind, n, motions, T=T, use_graphs=True)
    b = _driver(layout, kind, n, motions, T=T, use_graphs=False)
    s.refresh = lambda t, ws: None
    D = DOFS[layout]
    assert a.actions.shape == (n, T, D) and a.mus.shape == (n, T, D) and a.pd_tar.shape == (n, D) and a.z_actions is None
    assert a._sides()[1] is None
    _assert_same((a, s, b), "initial")
    resets = 0.0
    for use in ("eager", "capture", "replay"):
        for d in (a, s, b):
            d.play_steps()
        _assert_same((a, s, b), use)
        assert torch.equal(a.pd_tar, _pd_composition(a, T - 1)), f"{use}: pd_tar"
        resets += float(a.dones.sum())
        for d in (a, s, b):
            d.finish()
        assert all(torch.equal(a.adv, d.adv) and torch.equal(a.ret, d.ret) for d in (s, b))
    assert resets > 0 and bool(torch.isfinite(a.obses).all()) and bool(torch.isfinite(a.actions).all())
    assert isinstance(a._graphs[("horizon",)], torch.cuda.CUDAGraph)
    assert all(isinstance(s._graphs[(seg, t)], torch.cuda.CUDAGraph) for seg in ("reset", "act", "post") for t in range(T))
    # the PPO update: graph-captured minibatches, finite statistics, moved parameters
    p0 = a.policy.flat.params.clone()
    stats = a.train_epoch(mini_epochs=2, minibatch=n * T // 4).clone()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(stats).all()) and float(stats.abs().sum()) > 0
    assert not torch.equal(p0, a.policy.flat.params) and bool(torch.isfinite(a.policy.flat.params).all())
    # a replayed iteration makes no host synchronisation
    torch.cuda.set_sync_debug_mode("error")
    try:
        a.play_steps()
        a.finish()
        a.train_epoch(mini_epochs=2, minibatch=n * T // 4)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


@pytest.mark.parametrize("layout,kind", [("smpl", "speed"), ("smplx", "reach")])
def test_driver_with_discriminator(layout, kind, motions):
    """The baseline with the AMP part: graph equals eager over three iterations of play_steps, finish (task and discriminator rewards
    mixed) and train_epoch, and the parameters move."""
    N, T, MB = 24, 4, 32
    a = _driver(layout, kind, N, motions, T=T, use_graphs=True, amp=True, units=(256, 128))
    b = _driver(layout, kind, N, motions, T=T, use_graphs=False, amp=True, units=(256, 128))
    assert a.policy.disc is not None and a.policy.A == DOFS[layout]
    p0 = a.policy.flat.params.clone()
    for it in range(3):
        stats = []
        for x in (a, b):
            x.play_steps()
            x.finish()
            stats.append(x.train_epoch(mini_epochs=2, minibatch=MB).clone())
        _assert_same((a, b), f"iteration {it}")
        for k in ("adv", "ret"):
            assert torch.equal(getattr(a, k), getattr(b, k)), f"iteration {it}: {k}"
        assert torch.equal(a.policy.flat.params, b.policy.flat.params), f"iteration {it}: parameters"
        assert bool(torch.isfinite(stats[0]).all())
        assert torch.equal(a.pd_tar, _pd_composition(a, T - 1))
    assert not torch.equal(p0, a.policy.flat.params)
    assert bool(torch.isfinite(a.amp_obs).all()) and float(a.amp_obs.abs().sum()) > 0
