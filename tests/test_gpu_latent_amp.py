"""Discriminator training in the latent-space drivers (reach, speed, strike: ZTaskStepsB200; terrain: TerrainStepsB200; VR:
ImZStepsB200), each through its own reset's AMP path, and the demo fetch's rows.

Bars, per driver at a small env count:
  * amp_obs[:, t] against an eager composition on an [N, steps, W] buffer: the current row element-wise against the float64
    build_amp_observations_smpl of the state it reads (tests/reset_fp64.py), the history rows bit for bit as the shift of the
    previous rows, or of the reset's back-filled rows for the envs reset at step t;
  * the graph-captured iteration against the eager one bit for bit, update and buffers included;
  * train_epoch against train_minibatch called by hand with the AMP batches the numpy ring model (tests/amp_buffers_model.py)
    selects, at each minibatch's row offset: the same parameters bit for bit, so the discriminator's gradients are inside the clip;
  * with disc_reward_w 0.5 the returns of task_w * r + disc_w * disc.rewards(amp_obs).
The demo fetch: clip and start time word for word, every row element-wise against the float64 motion AMP row at t0 - k dt."""
import numpy as np
import pytest
import torch

from tests import amp_buffers_model as M
from tests import reset_fp64 as rf
from tests.helpers import exact_tables
from tests.philox_ref import philox4x32_10, u01
from tests.test_gpu_imz_rollout import _driver as imz_driver, ml  # noqa: F401  (module fixture)
from tests.test_gpu_terrain_rollout import _driver as terrain_driver, env  # noqa: F401  (module fixture)
from tests.test_gpu_ztask_rollout import _driver as ztask_driver, motion  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N, T, MB = 24, 4, 32
DT = float(np.float32(1.0 / 60.0) * 2)
KEYS = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "lengths", "num_frames", "dt", "length_starts")
# case: (driver, amp_width, upright)
CASES = {"reach": ("reach", 196, True), "speed": ("speed", 195, False), "strike": ("strike", 195, True), "terrain": ("terrain", 196, True),
         "vr": ("vr", 196, True)}


def _amp(ml, width, upright):
    from pulse_b200.amp_buffers import AmpBuffersB200
    return AmpBuffersB200(ml, num_steps=10, amp_width=width, upright=upright, demo_buffer_size=160, replay_buffer_size=120, batch_size=64,
                          keep_prob=0.5, minibatch_size=16, seed=2)


def _build(case, use_graphs, request, disc_w=0.0):
    """The case's driver with a discriminator and the AMP part, on the pieces of the existing test drivers."""
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.sept import SeptPolicy
    kind, width, upright = CASES[case]
    kw = dict(horizon=T, use_graphs=use_graphs, reset_seed=3, task_reward_w=0.5 if disc_w else 1.0, disc_reward_w=disc_w)
    disc = dict(with_disc=True, amp_obs_size=10 * width, disc_units=(256, 128), device=DEV, seed=0)
    if kind in ("reach", "speed", "strike"):
        from pulse_b200.ztask_reset import ZTaskResetB200
        from pulse_b200.ztask_rollout import ZTaskStepsB200
        ml, floor = request.getfixturevalue("motion")
        d0 = ztask_driver(kind, N, (ml, floor), T=T, use_graphs=use_graphs)
        reset = ZTaskResetB200(kind, ml, floor, upright=upright, amp_root_height_obs=width == 196)
        pol = PPOPolicy(obs_size=d0.task.obs_size, num_actions=32, units=(256, 128), act="silu", **disc)
        d = ZTaskStepsB200(d0.task, reset, pol, d0.vae, d0.sim, pd_offset=d0.pd[0], pd_scale=d0.pd[1], pd_freeze=d0.pd_freeze,
                           amp=_amp(ml, width, upright), **kw)
    elif kind == "terrain":
        from pulse_b200.terrain_rollout import TerrainStepsB200
        env = request.getfixturevalue("env")
        d0 = terrain_driver(env, N, T=T, use_graphs=use_graphs)
        pol = SeptPolicy(num_actions=32, **disc)
        d = TerrainStepsB200(d0.task, d0.reset, pol, d0.vae, d0.sim, pd_offset=d0.pd[0], pd_scale=d0.pd[1], pd_freeze=d0.pd_freeze,
                             amp=_amp(env["ml"], d0.reset.amp_width, d0.reset.upright), **kw)
    else:
        from pulse_b200.imz_rollout import ImZStepsB200
        mlt = request.getfixturevalue("ml")
        d0 = imz_driver(mlt, N, T=T, use_graphs=use_graphs)
        pol = PPOPolicy(obs_size=d0.comp.obs_size, num_actions=32, units=(256, 128), act="silu", logstd=-1.5, **disc)
        d = ImZStepsB200(d0.comp, pol, d0.vae, d0.sim, pd_offset=d0.pd[0], pd_scale=d0.pd[1], pd_freeze=d0.pd_freeze,
                         amp=_amp(mlt[0], 196, True), **kw)
    d.first_observation()
    return d


@pytest.mark.parametrize("case", list(CASES))
def test_amp_rows_equal_eager_composition(case, request):
    d = _build(case, False, request)
    W, S = d.amp.amp_width, d.amp.num_steps
    upright = d.amp.upright
    snaps = {}

    def refresh(t, ws):                              # after reset(t): the state the row of step t reads, the back-filled rows, the flags
        s = d.sim
        snaps[t] = (s["body_state"][:, :24].clone(), s["dof_pos"].clone(), s["dof_vel"].clone(), d.amp_init.clone(), d.amp_fresh.clone() != 0)

    d.refresh = refresh
    for it in range(2):
        H = d.amp_obs[:, T - 1].view(N, S, W).clone()                    # the row before the horizon
        d.play_steps()
        d.finish()
        d.train_epoch(mini_epochs=1, minibatch=MB)
        for t in range(T):
            body, dp, dv, init, fresh = snaps[t]
            got = d.amp_obs[:, t].view(N, S, W)
            rf.check_amp(None, f"{case} it {it} step {t} current row", got[:, 0], rf.state_amp_ref(body, dp, dv, upright))
            hist = torch.where(fresh[:, None, None], init[:, :S - 1], H[:, :S - 1])
            assert torch.equal(got[:, 1:], hist), f"{case} it {it} step {t}: history rows"
            H = torch.cat([got[:, :1], hist], 1)
        assert not (d.amp_fresh != 0).any()


@pytest.mark.parametrize("case", list(CASES))
def test_graph_equals_eager(case, request):
    a, b = _build(case, True, request), _build(case, False, request)
    for it in range(3):
        for d in (a, b):
            d.play_steps()
            d.finish()
            d.train_epoch(mini_epochs=2, minibatch=MB)
        for k in ("amp_obs", "amp_init", "amp_fresh", "obses", "rewards", "adv", "ret"):
            assert torch.equal(getattr(a, k), getattr(b, k)), f"{case} iteration {it}: {k}"
        for ra, rb in ((a.amp.demo, b.amp.demo), (a.amp.replay, b.amp.replay)):
            assert torch.equal(ra.rows, rb.rows) and torch.equal(ra.ctr, rb.ctr), f"{case} iteration {it}: rings"
        assert torch.equal(a.policy.flat.params, b.policy.flat.params), f"{case} iteration {it}: parameters"


def _model(ring):
    m = M.RingModel(ring.capacity, ring.seed)
    m.head, m.total, m.sample_head, m.perm_key, m.draws = (int(x) for x in ring.ctr[:5].tolist())
    return m


@pytest.mark.parametrize("case", list(CASES))
def test_train_epoch_equals_train_minibatch_by_hand(case, request):
    a, b = _build(case, False, request), _build(case, False, request)
    rows, take = N * T, min(16, MB)
    for it in range(2):                                              # empty replay ring (the agent's rows), then a filled one
        for d in (a, b):
            d.play_steps()
            d.finish()
        a.train_epoch(mini_epochs=2, minibatch=MB)
        amp, W = b.amp, b.amp.row_floats
        amp.update_demos()
        flat = b.amp_obs.view(rows, W)
        md, mr = _model(amp.demo), _model(amp.replay)
        demo = amp.demo.rows[torch.from_numpy(md.sample(rows)).to(DEV)]
        ri = mr.sample(rows)
        replay = flat.clone() if ri is None else amp.replay.rows[torch.from_numpy(ri).to(DEV)]
        for ring, m in ((amp.demo, md), (amp.replay, mr)):
            ring.ctr[:5] = torch.from_numpy(m.counters()).to(DEV)
        b.policy.reset_stats()
        for _ in range(2):
            for i in range(rows // MB):
                r0, r1 = i * MB, (i + 1) * MB
                b.policy.train_minibatch(b.obses.view(rows, -1)[r0:r1], b.actions.view(rows, -1)[r0:r1], b.neglogp.view(rows)[r0:r1],
                                         b.adv[r0:r1], b.ret[r0:r1], old_mu=b.mus.view(rows, -1)[r0:r1],
                                         amp=(flat[r0:r0 + take], replay[r0:r0 + take], demo[r0:r0 + take]))
        amp.store_replay(flat)
        assert torch.equal(a.policy.flat.params, b.policy.flat.params), f"{case} iteration {it}: parameters"
        assert torch.equal(a.policy.stats, b.policy.stats)
        # the discriminator's fp64 loss sums are accumulated by atomics in the GEMM epilogues, in an order that varies between runs
        torch.testing.assert_close(a.policy.disc.stats, b.policy.disc.stats, rtol=1e-9, atol=0)
        for ra, rb in ((a.amp.demo, b.amp.demo), (a.amp.replay, b.amp.replay)):
            assert torch.equal(ra.ctr, rb.ctr) and torch.equal(ra.rows, rb.rows), f"{case} iteration {it}: rings"


@pytest.mark.parametrize("case", list(CASES))
def test_reward_mix(case, request):
    from pulse_b200.rollout import discount_values
    d = _build(case, False, request, disc_w=0.5)
    d.play_steps()
    r = d.rewards.clone()
    disc_r = d.policy.disc.rewards(d.amp_obs.view(N * T, -1).clone()).view(N, T).t()
    d.finish()
    adv, _ = discount_values(d.dones, d.values, 0.5 * r.unsqueeze(-1) + 0.5 * disc_r.unsqueeze(-1), d.next_values, gamma=d.gamma, tau=d.tau,
                             normalize_advantage=True)
    assert torch.equal(d.adv, adv)
    assert disc_r.abs().sum() > 0


def test_refusals(request):
    from pulse_b200 import _lib
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    d = _build("speed", False, request)
    with pytest.raises(_lib.PulseError, match="discriminator"):
        ZTaskStepsB200(d.task, d.reset, d.policy, d.vae, d.sim, horizon=T)
    with pytest.raises(_lib.PulseError, match="at least 2 steps"):
        ZTaskStepsB200(d.task, d.reset, d.policy, d.vae, d.sim, horizon=1, amp=d.amp)


# ------------------------------------------------------------------------------------------------ the demo fetch's rows
@pytest.fixture(scope="module")
def demo_tables():
    from pulse_b200.motion_lib import MotionLibB200
    tb = exact_tables(23, seed=9, min_frames=4, spread=120)
    t = {k: getattr(tb, k).clone() for k in KEYS}
    return MotionLibB200.from_tables({k: getattr(tb, k) for k in KEYS + ("motion_aa",)}, device=DEV), t


@pytest.mark.parametrize("width,upright", [(196, True), (195, True), (196, False), (195, False)])
def test_demo_fetch_rows_fp64(demo_tables, width, upright):
    from pulse_b200.amp_buffers import AmpBuffersB200
    ml, t = demo_tables
    cap, B = 300, 128
    bufs = AmpBuffersB200(ml, num_steps=10, amp_width=width, upright=upright, demo_buffer_size=cap, batch_size=B, seed=4)
    mids = torch.empty(B, dtype=torch.int64, device=DEV)
    t0 = torch.empty(B, device=DEV)
    td = {k: v.to(DEV) for k, v in t.items()}
    i = np.arange(B)
    for it in range(3):                                              # the third fetch wraps the ring
        head = int(bufs.demo.ctr[0])
        bufs.fetch_demos(motion_ids_out=mids, times_out=t0)
        u = torch.from_numpy(u01(philox4x32_10(bufs.demo.seed, [(M.PLANE_DEMO_CLIP << 32) + k for k in i], it)[0]))
        want_ids = rf.pick_motion_ref(ml.sampling_cdf(), u)
        assert torch.equal(mids.cpu(), want_ids)
        ph = torch.from_numpy(u01(philox4x32_10(bufs.demo.seed, [(M.PLANE_DEMO_TIME << 32) + k for k in i], it)[0]))
        want_t0 = rf.start_time_ref(ph, t["lengths"][want_ids])
        assert torch.equal(t0.cpu(), want_t0)
        slots = torch.from_numpy((head + i) % cap).to(DEV)
        rows = bufs.demo.rows[slots].view(B, 10, width)
        times = rf.history_times(want_t0, DT, 10)
        for k in range(10):
            rf.check_amp(None, f"demo {width} upright {upright} fetch {it} row {k}", rows[:, k],
                         rf.motion_amp_ref(rf.motion_ref(td, want_ids.to(DEV), times[:, k].to(DEV)), upright))
    np.testing.assert_array_equal(bufs.demo.counters().cpu().numpy(), [(3 * B) % cap, 3 * B, 0, 0, 3])
