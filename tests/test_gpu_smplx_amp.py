"""The PULSE-X AMP path on the device (52-body SMPL-X humanoid, env_pulsex_amp.yaml): `pulse_smplx_amp_obs_row`, the AMP back-fill of
`pulse_reset_ztask_smplx`, `pulse_smplx_amp_demo_fetch` and the SMPL-X speed driver with a discriminator.

Bars:
  * the row kernel at 1, 300, 2051 and 16384 envs and both widths: the current row element-wise against the float64 row
    (tests/smplx_amp_fp64.py) and on the fixture's states against the reference's rows; the history bit for bit as the shift of the
    previous row, or the back-filled rows for fresh envs; the fresh flags cleared;
  * the reset: rows k >= 1 against the float64 motion row at t0 - k dt, row 0 against the state written; the state outputs and draws
    bit-identical to the same call without the AMP buffer; the reference fixture's recorded draws replayed;
  * the demo fetch: clips and start times word for word, every row against float64 at both widths, a third fetch that wraps the ring;
  * the driver: the four bars of test_gpu_latent_amp.py (rows against an eager composition, graph = eager bit for bit, train_epoch =
    train_minibatch by hand, the reward mix);
  * refusals of mismatched widths, layouts and upright settings."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import amp_buffers_model as M
from tests import reset_fp64 as rf
from tests import smplx_amp_fp64 as xf
from tests import smplx_speed_oracle as so
from tests.philox_ref import philox4x32_10, u01
from tests.test_gpu_smplx_speed import _driver as smplx_driver, motion  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = float(np.float32(1.0 / 60.0) * 2)
HERE = os.path.dirname(os.path.abspath(__file__))
N, T, MB = 24, 4, 32


def _golden():
    return np.load(os.path.join(HERE, "golden", "smplx_amp.npz"))


def _row_call(body, dof_state, prev, out, width, fresh=None, fresh_rows=None):
    from pulse_b200 import _lib
    lib = _lib.load()
    dp, dv = dof_state[:, :, 0], dof_state[:, :, 1]
    a = _lib.AmpRowArgs(body_state=body.data_ptr(), body_env_stride=body.stride(0), dof_pos=dp.data_ptr(), dof_vel=dv.data_ptr(),
                        dof_env_stride=dp.stride(0), dof_elem_stride=dp.stride(1), prev=prev.data_ptr(), ld_prev=prev.stride(0),
                        out=out.data_ptr(), ld_out=out.stride(0), num_steps=10, fresh=_lib.ptr(fresh), fresh_rows=_lib.ptr(fresh_rows),
                        amp_width=width, remove_base_rot=1)
    _lib.check(lib.pulse_smplx_amp_obs_row(C.byref(a), body.shape[0], _lib.current_stream(DEV)), "pulse_smplx_amp_obs_row")


@pytest.mark.parametrize("width", [465, 466])
@pytest.mark.parametrize("n", [1, 300, 2051, 16384])
def test_row_kernel(n, width):
    g = torch.Generator().manual_seed(n + width)
    body = torch.zeros(n, 53, 13)
    body[..., 0:3] = torch.randn(n, 53, 3, generator=g) * 0.4 + torch.tensor([0.0, 0.0, 0.9])
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 53, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 53, 6, generator=g)
    dof_state = torch.randn(n, 153, 2, generator=g)
    body, dof_state = body.to(DEV), dof_state.to(DEV)
    prev = torch.randn(n, 10 * width + 3, generator=g).to(DEV)[:, :10 * width]          # padded rows: ld_prev != 10 W
    out = torch.full((n, 10 * width), -3.0, device=DEV)
    fresh = (torch.rand(n, generator=g) < 0.3).int().to(DEV)
    fresh_rows = torch.randn(n, 10, width, generator=g).to(DEV)
    want_fresh = fresh.clone() != 0
    _row_call(body, dof_state, prev, out, width, fresh, fresh_rows)
    torch.cuda.synchronize()
    got = out.view(n, 10, width)
    xf.check_amp(None, f"row {n} {width}", got[:, 0], xf.state_amp_ref(body, dof_state[:, :, 0], dof_state[:, :, 1]))
    hist = torch.where(want_fresh[:, None, None], fresh_rows[:, :9], prev.reshape(n, 10, width)[:, :9])
    assert torch.equal(got[:, 1:], hist)
    assert int(fresh.abs().sum()) == 0
    assert bool(want_fresh.any()) or n == 1


@pytest.mark.parametrize("height", [True, False])
def test_row_kernel_on_fixture_states(height):
    from tests.test_smplx_amp_cpu import gen
    m, gd = gen(), _golden()
    bs, dof_pos, dof_vel = m.state_inputs()
    n, width = bs.shape[0], 466 if height else 465
    body = torch.zeros(n, 52, 13)
    body[:] = bs
    dof_state = torch.stack([dof_pos, dof_vel], -1).to(DEV)
    prev, out = torch.zeros(n, 10 * width, device=DEV), torch.zeros(n, 10 * width, device=DEV)
    _row_call(body.to(DEV), dof_state, prev, out, width)
    torch.cuda.synchronize()
    want = gd["state_amp"] if height else gd["state_amp"][:, 1:]              # the 465-float rows drop the root height
    torch.testing.assert_close(out[:, :width].cpu(), torch.from_numpy(np.ascontiguousarray(want)), atol=2e-5, rtol=2e-5)


# ------------------------------------------------------------------------------------------------ the reset's back-fill
def _reset_state(n, seed):
    g = torch.Generator().manual_seed(seed)
    st = dict(root_states=torch.randn(n, 13, generator=g), dof_pos=torch.randn(n, 153, generator=g), dof_vel=torch.randn(n, 153, generator=g),
              rigid_body_state=torch.randn(n, 53, 13, generator=g), sampled_motion_ids=torch.zeros(n, dtype=torch.int64),
              motion_start_times=torch.zeros(n), progress_buf=torch.randint(0, 300, (n,), generator=g),
              reset_buf=(torch.rand(n, generator=g) < 0.3).long(), terminate_buf=torch.ones(n, dtype=torch.int64),
              contact_forces=torch.randn(n, 53, 3, generator=g))
    return {k: v.to(DEV) for k, v in st.items()}


def _check_backfill(tb, st, ids, buf, width):
    """Rows k >= 1 of the reset envs against the float64 motion at t0 - k dt, row 0 against the state written."""
    td = {k: v.to(DEV) for k, v in so.table_dict(tb).items()}
    mids, t0 = st["sampled_motion_ids"][ids], st["motion_start_times"][ids]
    times = rf.history_times(t0.cpu(), DT, 10).to(DEV)
    for k in range(1, 10):
        xf.check_amp(None, f"reset row {k}", buf[ids, k], xf.motion_amp_ref(rf.motion_ref(td, mids, times[:, k])))
    xf.check_amp(None, "reset row 0", buf[ids, 0], xf.state_amp_ref(st["rigid_body_state"][ids], st["dof_pos"][ids], st["dof_vel"][ids]))


@pytest.mark.parametrize("draws", ["injected", "philox"])
@pytest.mark.parametrize("width", [465, 466])
def test_reset_backfill(motion, width, draws):
    from pulse_b200.ztask_reset import ZTaskResetB200
    tb, ml, floor = motion
    n = 2051
    r = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False, amp_root_height_obs=width == 466)
    assert r.amp_width == width
    g = torch.Generator().manual_seed(9)
    kw = dict(motion_u=torch.rand(n, generator=g).to(DEV), phase=torch.rand(n, generator=g).to(DEV)) if draws == "injected" else {}
    plain, st = _reset_state(n, 11), _reset_state(n, 11)
    buf = torch.full((n, 10, width), 7.0, device=DEV)
    fresh = torch.zeros(n, dtype=torch.int32, device=DEV)
    ws0 = r.reset_envs(**plain, seed=4, offset=2, **kw)
    cnt0, list0 = int(ws0["count"].item()), ws0["env_list"].clone()
    ws = r.reset_envs(**st, amp_obs_buf=buf, amp_fresh=fresh, seed=4, offset=2, **kw)
    torch.cuda.synchronize()
    assert int(ws["count"].item()) == cnt0 > 0 and torch.equal(ws["env_list"][:cnt0], list0[:cnt0])
    for k in plain:
        assert torch.equal(plain[k], st[k]), f"{k}: the AMP buffer changed the reset's state outputs"
    ids = list0[:cnt0]
    keep = torch.ones(n, dtype=torch.bool, device=DEV)
    keep[ids] = False
    assert bool((buf[keep] == 7.0).all()) and torch.equal(fresh != 0, ~keep)
    _check_backfill(tb, st, ids, buf, width)


def test_reset_backfill_replays_the_reference_fixture():
    """The draws the reference's HumanoidSpeed reset recorded (tests/golden/smplx_speed.npz), replayed with the AMP buffer: the state
    within the speed fixture's bounds, the back-filled rows against float64."""
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ztask_reset import ZTaskResetB200
    from tests.test_gpu_smplx_speed import gen
    from tests.test_smplx_speed_cpu import reset_draws, reset_tables
    m = gen()
    g = np.load(os.path.join(HERE, "golden", "smplx_speed.npz"))
    n = m.RESET_N
    ids, d = reset_draws(g, n)
    tb, floor = reset_tables(m)
    ml = MotionLibB200.from_tables(so.table_dict(tb), device=DEV)
    ml._sampling_batch_prob = torch.from_numpy(g["r_prob"]).to(DEV)
    r = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False)
    z = lambda *s, **k: torch.zeros(*s, device=DEV, **k)
    st = dict(root_states=z(n, 13), dof_pos=z(n, 153), dof_vel=z(n, 153), rigid_body_state=z(n, 53, 13),
              progress_buf=torch.ones(n, dtype=torch.int64, device=DEV), sampled_motion_ids=z(n, dtype=torch.int64), motion_start_times=z(n))
    buf = z(n, 10, 465)
    r.reset_envs(**st, env_ids=ids.to(DEV), motion_ids=d["motion_ids"].to(DEV), phase=d["phase"].to(DEV), amp_obs_buf=buf)
    torch.cuda.synchronize()
    T_ = lambda k: torch.from_numpy(g[k])[ids]
    assert torch.equal(st["sampled_motion_ids"].cpu()[ids], T_("r_motion_ids")) and torch.equal(st["motion_start_times"].cpu()[ids], T_("r_start_times"))
    torch.testing.assert_close(st["rigid_body_state"].cpu()[ids, :52], T_("r_body_state"), atol=2e-5, rtol=0)
    torch.testing.assert_close(st["dof_pos"].cpu()[ids], T_("r_dof_pos"), atol=2e-5, rtol=0)
    _check_backfill(tb, st, ids.to(DEV), buf, 465)


# ------------------------------------------------------------------------------------------------ the demo fetch
@pytest.fixture(scope="module")
def demo_tables():
    from pulse_b200.motion_lib import MotionLibB200
    tb = so.tables(23, seed=9, min_frames=4, spread=120)
    return MotionLibB200.from_tables(so.table_dict(tb), device=DEV), tb


@pytest.mark.parametrize("width", [465, 466])
def test_demo_fetch_rows_fp64(demo_tables, width):
    from pulse_b200.amp_buffers import AmpBuffersB200
    ml, tb = demo_tables
    cap, B = 300, 128
    bufs = AmpBuffersB200(ml, num_steps=10, amp_width=width, upright=False, demo_buffer_size=cap, batch_size=B, seed=4)
    mids = torch.empty(B, dtype=torch.int64, device=DEV)
    t0 = torch.empty(B, device=DEV)
    td = {k: v.to(DEV) for k, v in so.table_dict(tb).items()}
    i = np.arange(B)
    for it in range(3):                                              # the third fetch wraps the ring
        head = int(bufs.demo.ctr[0])
        bufs.fetch_demos(motion_ids_out=mids, times_out=t0)
        u = torch.from_numpy(u01(philox4x32_10(bufs.demo.seed, [(M.PLANE_DEMO_CLIP << 32) + k for k in i], it)[0]))
        want_ids = rf.pick_motion_ref(ml.sampling_cdf(), u)
        assert torch.equal(mids.cpu(), want_ids)
        ph = torch.from_numpy(u01(philox4x32_10(bufs.demo.seed, [(M.PLANE_DEMO_TIME << 32) + k for k in i], it)[0]))
        want_t0 = rf.start_time_ref(ph, tb.lengths[want_ids])
        assert torch.equal(t0.cpu(), want_t0)
        slots = torch.from_numpy((head + i) % cap).to(DEV)
        rows = bufs.demo.rows[slots].view(B, 10, width)
        times = rf.history_times(want_t0, DT, 10)
        for k in range(10):
            xf.check_amp(None, f"demo {width} fetch {it} row {k}", rows[:, k],
                         xf.motion_amp_ref(rf.motion_ref(td, want_ids.to(DEV), times[:, k].to(DEV))))
    np.testing.assert_array_equal(bufs.demo.counters().cpu().numpy(), [(3 * B) % cap, 3 * B, 0, 0, 3])


# ------------------------------------------------------------------------------------------------ the driver
def _build(motion, use_graphs, disc_w=0.0, width=465):
    from pulse_b200.amp_buffers import AmpBuffersB200
    from pulse_b200.ppo import PPOPolicy
    from pulse_b200.ztask_reset import ZTaskResetB200
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    _, ml, floor = motion
    d0 = smplx_driver(N, motion, T=T, use_graphs=use_graphs)
    reset = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False, amp_root_height_obs=width == 466)
    pol = PPOPolicy(obs_size=781, num_actions=48, units=(256, 128), act="silu", with_disc=True, amp_obs_size=10 * width, disc_units=(256, 128),
                    device=DEV, seed=0)
    amp = AmpBuffersB200(ml, num_steps=10, amp_width=width, upright=False, demo_buffer_size=160, replay_buffer_size=120, batch_size=64,
                         keep_prob=0.5, minibatch_size=16, seed=2)
    d = ZTaskStepsB200(d0.task, reset, pol, d0.vae, d0.sim, horizon=T, pd_offset=d0.pd[0], pd_scale=d0.pd[1], use_graphs=use_graphs,
                       reset_seed=3, amp=amp, task_reward_w=0.5 if disc_w else 1.0, disc_reward_w=disc_w)
    d.first_observation()
    return d


@pytest.mark.parametrize("width", [465, 466])
def test_driver_amp_rows_equal_eager_composition(motion, width):
    d = _build(motion, False, width=width)
    W, S = d.amp.amp_width, d.amp.num_steps
    snaps = {}

    def refresh(t, ws):
        s = d.sim
        snaps[t] = (s["body_state"][:, :52].clone(), s["dof_pos"].clone(), s["dof_vel"].clone(), d.amp_init.clone(), d.amp_fresh.clone() != 0)

    d.refresh = refresh
    fresh_seen = 0
    for it in range(2):
        H = d.amp_obs[:, T - 1].view(N, S, W).clone()
        d.play_steps()
        d.finish()
        d.train_epoch(mini_epochs=1, minibatch=MB)
        for t in range(T):
            body, dp, dv, init, fresh = snaps[t]
            fresh_seen += int(fresh.sum())
            got = d.amp_obs[:, t].view(N, S, W)
            xf.check_amp(None, f"smplx it {it} step {t} current row", got[:, 0], xf.state_amp_ref(body, dp, dv))
            hist = torch.where(fresh[:, None, None], init[:, :S - 1], H[:, :S - 1])
            assert torch.equal(got[:, 1:], hist), f"it {it} step {t}: history rows"
            H = torch.cat([got[:, :1], hist], 1)
        assert not (d.amp_fresh != 0).any()
    assert fresh_seen > 0


def test_driver_graph_equals_eager(motion):
    a, b = _build(motion, True), _build(motion, False)
    for it in range(3):
        for d in (a, b):
            d.play_steps()
            d.finish()
            d.train_epoch(mini_epochs=2, minibatch=MB)
        for k in ("amp_obs", "amp_init", "amp_fresh", "obses", "rewards", "adv", "ret"):
            assert torch.equal(getattr(a, k), getattr(b, k)), f"iteration {it}: {k}"
        for ra, rb in ((a.amp.demo, b.amp.demo), (a.amp.replay, b.amp.replay)):
            assert torch.equal(ra.rows, rb.rows) and torch.equal(ra.ctr, rb.ctr), f"iteration {it}: rings"
        assert torch.equal(a.policy.flat.params, b.policy.flat.params), f"iteration {it}: parameters"


def _model(ring):
    m = M.RingModel(ring.capacity, ring.seed)
    m.head, m.total, m.sample_head, m.perm_key, m.draws = (int(x) for x in ring.ctr[:5].tolist())
    return m


def test_driver_train_epoch_equals_train_minibatch_by_hand(motion):
    a, b = _build(motion, False), _build(motion, False)
    rows, take = N * T, min(16, MB)
    for it in range(2):
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
        assert torch.equal(a.policy.flat.params, b.policy.flat.params), f"iteration {it}: parameters"
        assert torch.equal(a.policy.stats, b.policy.stats)
        torch.testing.assert_close(a.policy.disc.stats, b.policy.disc.stats, rtol=1e-9, atol=0)
        for ra, rb in ((a.amp.demo, b.amp.demo), (a.amp.replay, b.amp.replay)):
            assert torch.equal(ra.ctr, rb.ctr) and torch.equal(ra.rows, rb.rows), f"iteration {it}: rings"


def test_driver_reward_mix(motion):
    from pulse_b200.rollout import discount_values
    d = _build(motion, False, disc_w=0.5)
    d.play_steps()
    r = d.rewards.clone()
    disc_r = d.policy.disc.rewards(d.amp_obs.view(N * T, -1).clone()).view(N, T).t()
    d.finish()
    adv, _ = discount_values(d.dones, d.values, 0.5 * r.unsqueeze(-1) + 0.5 * disc_r.unsqueeze(-1), d.next_values, gamma=d.gamma, tau=d.tau,
                             normalize_advantage=True)
    assert torch.equal(d.adv, adv)
    assert disc_r.abs().sum() > 0


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(motion):
    from pulse_b200 import PulseError
    from pulse_b200.amp_buffers import AmpBuffersB200
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ztask_reset import ZTaskResetB200, check_amp_layout
    from pulse_b200.ztask_rollout import ZTaskStepsB200
    from tests.helpers import exact_tables
    _, ml, floor = motion
    d = _build(motion, False)
    for width, upright, what in ((196, False, "465"), (195, False, "465"), (465, True, "upright=False")):
        with pytest.raises(PulseError, match=what):
            AmpBuffersB200(ml, amp_width=width, upright=upright)
    tb = exact_tables(5, seed=3, min_frames=4, spread=20)
    keys = ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "lengths", "num_frames", "dt", "length_starts", "motion_aa")
    ml24 = MotionLibB200.from_tables({k: getattr(tb, k) for k in keys}, device=DEV)
    for width in (465, 466):
        with pytest.raises(PulseError, match="195"):
            AmpBuffersB200(ml24, amp_width=width, upright=False)
    smpl_amp = AmpBuffersB200(ml24, amp_width=195, upright=False, demo_buffer_size=16, replay_buffer_size=16, batch_size=8)
    with pytest.raises(PulseError, match="AMP part"):                  # SMPL rows under the SMPL-X driver
        ZTaskStepsB200(d.task, d.reset, d.policy, d.vae, d.sim, horizon=T, amp=smpl_amp)
    r466 = ZTaskResetB200("speed", ml, floor.to(DEV), upright=False, amp_root_height_obs=True)
    with pytest.raises(PulseError, match="AMP part"):                  # 465-float AMP part, 466-float reset
        ZTaskStepsB200(d.task, r466, d.policy, d.vae, d.sim, horizon=T, amp=d.amp)
    with pytest.raises(PulseError, match="discriminator reads"):       # a discriminator of the SMPL width
        from pulse_b200.ppo import PPOPolicy
        pol = PPOPolicy(obs_size=781, num_actions=48, units=(256, 128), act="silu", with_disc=True, amp_obs_size=1950, disc_units=(256, 128),
                        device=DEV, seed=0)
        ZTaskStepsB200(d.task, d.reset, pol, d.vae, d.sim, horizon=T, amp=d.amp)
    with pytest.raises(PulseError, match="SMPL-X"):                    # the SMPL entry points never get the SMPL-X handle
        ml.handle
    with pytest.raises(PulseError, match="no SMPL-X handle"):
        ml24.smplx_handle
    n = 8
    z = lambda *s, **k: torch.zeros(*s, device=DEV, **k)
    kw = dict(root_states=z(n, 13), dof_pos=z(n, 153), dof_vel=z(n, 153), rigid_body_state=z(n, 52, 13), progress_buf=z(n, dtype=torch.int64),
              sampled_motion_ids=z(n, dtype=torch.int64), motion_start_times=z(n), reset_buf=z(n, dtype=torch.int64))
    with pytest.raises(PulseError, match="465"):
        d.reset.reset_envs(**kw, amp_obs_buf=z(n, 10, 195))
    from types import SimpleNamespace as NS
    task = NS(amp_obs_v=1, _key_body_ids=torch.tensor([7, 3, 22, 17]), dof_subset=torch.arange(153), _has_dof_subset=True)
    with pytest.raises(PulseError, match="keyBodies"):
        check_amp_layout(task, "PULSE-X", smplx=True)
    task._key_body_ids = torch.tensor([7, 3, 36, 17])
    with pytest.raises(PulseError, match="dof_subset"):
        check_amp_layout(task, "PULSE-X", smplx=True)
