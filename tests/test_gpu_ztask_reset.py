"""Reference-state reset of the latent-space tasks (`pulse_reset_ztask`, `pulse_ztask_reset_task` through
`pulse_b200.ztask_reset.ZTaskResetB200`) against the CPU oracle tests/ztask_reset_oracle.py, which tests/test_ztask_reset_cpu.py pins
to the unmodified reference.

Bars (those of test_gpu_reset.py): env / actor / target-actor lists, counts, clips, start times, counters and change steps bit-exact;
simulator tensors within 1e-5 (bodies also rtol 2e-5), dof positions and AMP rows within 1e-4; every env that is not reset and every
buffer the task does not own bit-identical.  Philox draws: clip frequencies against the sampling weights (chi-square, zero-weight clips
never drawn), start phases, the strike near fraction and the task draws; CUDA-graph replay with a device-side offset equals eager."""
import pytest
import torch

from tests import ztask_reset_oracle as zo
from tests.helpers import exact_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIPS = 23


@pytest.fixture(scope="module")
def env():
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.ztask_reset import smpl_ground_table
    tb = exact_tables(CLIPS, seed=9, min_frames=4, spread=120)
    betas = torch.linspace(-1.0, 1.0, 10)
    floor = smpl_ground_table(tb.motion_aa, zo.StandInParser(), betas)
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames",
                                                                 "dt", "length_starts")}, device=DEV)
    prob = torch.rand(CLIPS, generator=torch.Generator().manual_seed(4))
    prob[[1, 5, 11]] = 0.0
    ml._sampling_batch_prob = (prob / prob.sum()).to(DEV)
    return tb, ml, floor


def _make(kind, env, upright=True, state_init="Random"):
    from pulse_b200.ztask_reset import ZTaskResetB200
    tb, ml, floor = env
    return ZTaskResetB200(kind, ml, floor.to(DEV), upright=upright, state_init=state_init)


def _state(n, seed):
    """Oracle-side state (dense CPU) and Isaac-Gym shaped device tensors: 2 actors per env, 72 dofs x (pos, vel), 26 bodies, with
    padding 5.0 the reset must not touch."""
    g = torch.Generator().manual_seed(seed)
    st = {"root_states": torch.randn(n, 13, generator=g), "dof_pos": torch.randn(n, 69, generator=g), "dof_vel": torch.randn(n, 69, generator=g),
          "body_state": torch.randn(n, 24, 13, generator=g), "sampled_motion_ids": torch.randint(0, CLIPS, (n,), generator=g),
          "motion_start_times": torch.rand(n, generator=g), "progress_buf": torch.randint(0, 300, (n,), generator=g),
          "reset_buf": torch.zeros(n, dtype=torch.int64), "terminate_buf": (torch.rand(n, generator=g) < 0.3).long(),
          "contact_forces": torch.randn(n, 26, 3, generator=g), "amp_obs_buf": torch.randn(n, 10, 195, generator=g),
          "target_states": torch.randn(n, 13, generator=g)}
    d = {k: st[k].to(DEV).clone() for k in ("sampled_motion_ids", "motion_start_times", "progress_buf", "reset_buf", "terminate_buf", "amp_obs_buf")}
    d["root_all"] = torch.full((n, 2, 13), 5.0, device=DEV)
    d["root_all"][:, 0], d["root_all"][:, 1] = st["root_states"].to(DEV), st["target_states"].to(DEV)
    d["dof_state"] = torch.full((n, 72, 2), 5.0, device=DEV)
    d["dof_state"][:, :69, 0], d["dof_state"][:, :69, 1] = st["dof_pos"].to(DEV), st["dof_vel"].to(DEV)
    d["body"] = torch.full((n, 26, 13), 5.0, device=DEV)
    d["body"][:, :24] = st["body_state"].to(DEV)
    d["contact"] = st["contact_forces"].to(DEV).clone()
    d["actor_ids"] = torch.arange(n, dtype=torch.int32, device=DEV) * 2
    d["tar_actor_ids"] = d["actor_ids"] + 1
    return st, d


def _draws(n, seed, prob):
    g = torch.Generator().manual_seed(seed)
    return {"motion_ids": torch.multinomial(prob.cpu(), n, replacement=True, generator=g), "phase": torch.rand(n, generator=g),
            "strike_u": torch.rand(n, 4, generator=g), "task_u3": torch.rand(n, 3, generator=g), "task_u": torch.rand(n, generator=g),
            "steps": torch.randint(100, 200, (n,), generator=g)}


def _reset(r, d, kind, env_ids=None, draws=None, **kw):
    inj = {} if draws is None else {"motion_ids": draws["motion_ids"].to(DEV), "phase": draws["phase"].to(DEV),
                                    "strike_u": draws["strike_u"].to(DEV) if kind == "strike" else None}
    return r.reset_envs(root_states=d["root_all"][:, 0], dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1],
                        rigid_body_state=d["body"], progress_buf=d["progress_buf"], sampled_motion_ids=d["sampled_motion_ids"],
                        motion_start_times=d["motion_start_times"], reset_buf=None if env_ids is not None else d["reset_buf"], env_ids=env_ids,
                        terminate_buf=d["terminate_buf"], contact_forces=d["contact"], amp_obs_buf=d["amp_obs_buf"], actor_ids=d["actor_ids"],
                        target_states=d["root_all"][:, 1] if kind == "strike" else None, tar_actor_ids=d["tar_actor_ids"], **inj, **kw)


def _compare(d, exp, ids, n, kind, padding=True):
    close = lambda a, b, **k: torch.testing.assert_close(a.cpu(), b, **({"atol": 1e-5, "rtol": 0} | k))
    for k in ("sampled_motion_ids", "progress_buf", "reset_buf", "terminate_buf"):
        assert torch.equal(d[k].cpu(), exp[k]), k
    assert torch.equal(d["motion_start_times"].cpu(), exp["motion_start_times"])   # index arithmetic: bit-exact
    close(d["root_all"][:, 0], exp["root_states"])
    close(d["dof_state"][:, :69, 0], exp["dof_pos"], atol=1e-4, rtol=1e-4)
    close(d["dof_state"][:, :69, 1], exp["dof_vel"])
    close(d["body"][:, :24], exp["body_state"], rtol=2e-5)
    close(d["amp_obs_buf"], exp["amp_obs_buf"], atol=1e-4)
    assert torch.equal(d["contact"].cpu(), exp["contact_forces"])
    if kind == "strike":
        close(d["root_all"][:, 1], exp["target_states"], atol=2e-5)
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids] = False
    # padding (extra dofs / bodies) always, the target actor of the other tasks, and every env that was not reset: bit for bit
    if padding:
        assert float((d["dof_state"][:, 69:] - 5.0).abs().max()) == 0 and float((d["body"][:, 24:] - 5.0).abs().max()) == 0
    if kind != "strike":
        assert torch.equal(d["root_all"][:, 1].cpu(), exp["target_states"])
    for ours, ref in ((d["root_all"][:, 0], exp["root_states"]), (d["root_all"][:, 1], exp["target_states"]), (d["body"][:, :24], exp["body_state"]),
                      (d["amp_obs_buf"], exp["amp_obs_buf"]), (d["dof_state"][:, :69, 0], exp["dof_pos"]), (d["dof_state"][:, :69, 1], exp["dof_vel"])):
        assert torch.equal(ours.cpu()[keep], ref[keep])


def _check_lists(ws, ids, kind):
    cnt = int(ws["count"].item())
    assert cnt == ids.numel()
    assert torch.equal(ws["env_list"][:cnt].cpu(), ids)
    assert torch.equal(ws["actor_list"][:cnt].cpu(), (2 * ids).int())
    if kind == "strike":
        assert torch.equal(ws["tar_actor_list"][:cnt].cpu(), (2 * ids + 1).int())


CASES = [("reach", True, "Random"), ("speed", True, "Random"), ("speed", False, "Random"), ("strike", True, "Random"), ("speed", True, "Start"),
         ("strike", True, "Start")]


@pytest.mark.parametrize("n,frac,mode", [(257, 0.3, "mask"), (257, 0.3, "list"), (16384, 0.05, "mask"), (16384, 0.05, "list"), (16384, 1.0, "mask")])
@pytest.mark.parametrize("kind,upright,init", CASES)
def test_reset_matches_oracle(env, n, frac, mode, kind, upright, init):
    tb, ml, floor = env
    r = _make(kind, env, upright, init)
    st, d = _state(n, seed=n + len(kind))
    ids = (torch.rand(n, generator=torch.Generator().manual_seed(7)) < frac).nonzero().flatten()
    dr = _draws(n, 8, ml._sampling_batch_prob)
    if mode == "mask":
        d["reset_buf"][ids.to(DEV)] = 1
        st["reset_buf"][ids] = 1
        ws = _reset(r, d, kind, draws=dr)
    else:
        ws = _reset(r, d, kind, env_ids=ids.to(DEV), draws=dr)
    exp = zo.ztask_reset(tb, st, ids, dr, floor, kind, upright=upright, state_init=zo.RANDOM if init == "Random" else zo.START, width=195)
    torch.cuda.synchronize()
    _check_lists(ws, ids, kind)
    _compare(d, exp, ids, n, kind)
    if kind == "strike":
        return
    # _reset_task over the same list, injected draws: bit-exact
    chg = torch.randint(0, 500, (n,), device=DEV)
    chg0 = chg.cpu().clone()
    if kind == "reach":
        tar = torch.randn(n, 3, device=DEV)
        tar0 = tar.cpu().clone()
        r.reset_task(progress_buf=d["progress_buf"], change_steps=chg, tar_pos=tar, rand=dr["task_u3"].to(DEV), steps=dr["steps"].to(DEV))
        want, wchg = zo.reach_task(dr["task_u3"][ids], dr["steps"][ids], exp["progress_buf"][ids], **zo.REACH)
    else:
        tar = torch.randn(n, device=DEV)
        tar0 = tar.cpu().clone()
        r.reset_task(progress_buf=d["progress_buf"], change_steps=chg, tar_speed=tar, rand=dr["task_u"].to(DEV), steps=dr["steps"].to(DEV))
        want, wchg = zo.speed_task(dr["task_u"][ids], dr["steps"][ids], exp["progress_buf"][ids], **zo.SPEED)
    tar0[ids], chg0[ids] = want, wchg
    assert torch.equal(tar.cpu(), tar0) and torch.equal(chg.cpu(), chg0)


def test_empty_and_amp_width_196(env):
    """An empty id list touches nothing; the 196-float rows carry the root height in front of the 195-float layout."""
    tb, ml, floor = env
    from pulse_b200.ztask_reset import ZTaskResetB200
    n = 64
    st, d = _state(n, seed=1)
    before = {k: v.clone() for k, v in d.items()}
    ws = _reset(_make("reach", env), d, "reach", env_ids=torch.zeros(0, dtype=torch.int64, device=DEV))
    assert int(ws["count"].item()) == 0 and all(torch.equal(before[k], d[k]) for k in d)
    r196 = ZTaskResetB200("reach", ml, floor.to(DEV), amp_root_height_obs=True)
    ids = torch.arange(0, n, 3)
    dr = _draws(n, 2, ml._sampling_batch_prob)
    d["amp_obs_buf"] = torch.zeros(n, 10, 196, device=DEV)
    _reset(r196, d, "reach", env_ids=ids.to(DEV), draws=dr)
    st["amp_obs_buf"] = torch.zeros(n, 10, 196)
    exp = zo.ztask_reset(tb, st, ids, dr, floor, "reach", width=196)
    torch.testing.assert_close(d["amp_obs_buf"].cpu(), exp["amp_obs_buf"], atol=1e-4, rtol=0)
    assert float(d["amp_obs_buf"][ids, :, 0].abs().min()) > 0         # the root height leads the row
    with pytest.raises(Exception, match="amp_obs_buf"):
        _reset(_make("reach", env), d, "reach", env_ids=ids.to(DEV), draws=dr)


def test_philox_draw_statistics(env):
    """All 16384 envs reset with the kernel's own draws: clip frequencies follow the sampling weights (chi-square, zero-weight clips
    never drawn), start phases are uniform, the strike near fraction is near_prob, the task draws cover their ranges.  Same seed and
    offset -> the same draws; another offset -> other draws."""
    from scipy import stats
    tb, ml, floor = env
    n = 16384
    r = _make("strike", env)
    st, d = _state(n, seed=5)
    ws = _reset(r, d, "strike", env_ids=torch.arange(n, device=DEV), seed=1234, offset=77)
    ids = d["sampled_motion_ids"].cpu()
    prob = ml._sampling_batch_prob.cpu().double()
    counts = torch.bincount(ids, minlength=CLIPS).double()
    assert float(counts[prob == 0].sum()) == 0
    pos = prob > 0
    chi = stats.chisquare(counts[pos].numpy(), (prob[pos] / prob[pos].sum() * n).numpy())
    assert chi.pvalue > 1e-3, chi
    # start phases on the clips of 2 s and more, where the 1/30 s grid of sample_time_interval is fine: centred on the grid cell
    long = tb.num_frames[ids] >= 61
    ph = (d["motion_start_times"].cpu()[long] + 1.0 / 60.0) / tb.lengths[ids][long]
    assert int(long.sum()) > 2000 and float(ph.min()) > 0 and float(ph.max()) < 1.01
    assert abs(float(ph.mean()) - 0.5) < 0.02
    for q in (0.25, 0.5, 0.75):
        assert abs(float((ph < q).double().mean()) - q) < 0.03
    rel = d["root_all"][:, 1, :2].cpu() - d["root_all"][:, 0, :2].cpu()
    near = float((rel.norm(dim=-1) <= zo.STRIKE["near_dist"] + 1e-4).double().mean())
    # near envs always land within near_dist; far ones only with probability (1.5 - 0.5) / (10 - 0.5)
    expect = zo.STRIKE["near_prob"] + (1 - zo.STRIKE["near_prob"]) * (1.0 / 9.5)
    assert abs(near - expect) < 0.02, near
    first = d["sampled_motion_ids"].clone()
    _reset(r, d, "strike", env_ids=torch.arange(n, device=DEV), seed=1234, offset=77)
    assert torch.equal(first, d["sampled_motion_ids"])
    _reset(r, d, "strike", env_ids=torch.arange(n, device=DEV), seed=1234, offset=78)
    assert not torch.equal(first, d["sampled_motion_ids"])
    # reach task draws
    rr = _make("reach", env)
    _reset(rr, d, "reach", env_ids=torch.arange(n, device=DEV), seed=5)
    tar, chg = torch.zeros(n, 3, device=DEV), torch.zeros(n, dtype=torch.int64, device=DEV)
    rr.reset_task(progress_buf=d["progress_buf"], change_steps=chg, tar_pos=tar, seed=5)
    tar, chg = tar.cpu(), chg.cpu()
    assert float(tar[:, :2].abs().max()) <= 1.0 and 0.5 <= float(tar[:, 2].min()) and float(tar[:, 2].max()) < 1.5
    assert int(chg.min()) == 100 and int(chg.max()) == 199 and abs(float(chg.double().mean()) - 149.5) < 1.0
    assert abs(float(tar[:, 0].mean())) < 0.03 and abs(float(tar[:, 2].mean()) - 1.0) < 0.01


def test_cuda_graph_replay_equals_eager(env):
    """The reset and the task draw captured in one CUDA graph with a device-side offset: each replay equals the eager call at that
    offset."""
    n = 4096
    r = _make("reach", env)
    st, d = _state(n, seed=11)
    d["reset_buf"][::7] = 1
    init = {k: v.clone() for k, v in d.items()}
    tar, chg = torch.zeros(n, 3, device=DEV), torch.zeros(n, dtype=torch.int64, device=DEV)
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                       # warm-up outside the capture (workspace allocation)
        _reset(r, d, "reach", seed=3, offset_dev=off)
        r.reset_task(progress_buf=d["progress_buf"], change_steps=chg, tar_pos=tar, seed=3, offset_dev=off)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _reset(r, d, "reach", seed=3, offset_dev=off)
        r.reset_task(progress_buf=d["progress_buf"], change_steps=chg, tar_pos=tar, seed=3, offset_dev=off)
    for k in d:
        d[k].copy_(init[k])
    off.fill_(5)
    g.replay()
    torch.cuda.synchronize()
    got = {k: v.clone() for k, v in d.items()}
    got_tar, got_chg = tar.clone(), chg.clone()
    e = {k: v.clone() for k, v in init.items()}
    tar2, chg2 = torch.zeros(n, 3, device=DEV), torch.zeros(n, dtype=torch.int64, device=DEV)
    _reset(r, e, "reach", seed=3, offset=5)
    r.reset_task(progress_buf=e["progress_buf"], change_steps=chg2, tar_pos=tar2, seed=3, offset=5)
    torch.cuda.synchronize()
    for k in got:
        assert torch.equal(got[k], e[k]), k
    assert torch.equal(got_tar[::7], tar2[::7]) and torch.equal(got_chg[::7], chg2[::7])


def test_sampling_cdf_follows_the_probabilities(env):
    tb, ml, floor = env
    c0 = ml.sampling_cdf()
    assert ml.sampling_cdf() is c0                                 # cached while the weights stand
    ml._sampling_batch_prob[0] += 0.0                              # an in-place change bumps the version: rebuilt
    assert ml.sampling_cdf() is not c0
    torch.testing.assert_close(ml.sampling_cdf().cpu(), torch.cumsum(ml._sampling_batch_prob.cpu(), 0))


@pytest.mark.parametrize("kind", ["reach", "speed", "strike"])
def test_list_observation_equals_the_full_step(kind):
    """pulse_reach_obs_list / pulse_ztask_obs_list write, for the listed envs, the rows the full step kernel writes, bit for bit, and
    touch nothing else: other rows, reward, reset and terminate words stay."""
    from pulse_b200.reach import ReachTaskB200
    from pulse_b200.ztasks import SpeedTaskB200, StrikeTaskB200
    n = 3001
    g = torch.Generator().manual_seed(21)
    body = (torch.randn(n, 26, 13, generator=g) * 0.5).to(DEV)
    body[:, :, 3:7] /= body[:, :, 3:7].norm(dim=-1, keepdim=True)
    progress = torch.randint(0, 300, (n,), generator=g).to(DEV)
    target = torch.randn(n, 13, generator=g).to(DEV)
    tar_contact = torch.randn(n, 3, generator=g).to(DEV)
    mk = {"reach": ReachTaskB200, "speed": SpeedTaskB200, "strike": StrikeTaskB200}[kind]
    full, part = mk(n, device=DEV), mk(n, device=DEV)
    for t in (full, part):
        if kind == "reach":
            t._tar_pos.copy_(torch.randn(n, 3, generator=torch.Generator().manual_seed(1)).to(DEV))
        if kind == "speed":
            t._tar_speed.copy_(torch.rand(n, generator=torch.Generator().manual_seed(1)).to(DEV) * 4)
    if kind == "strike":
        full.post_physics_step(body, progress, target, tar_contact)
    else:
        full.post_physics_step(body, progress)
    part.obs_buf.fill_(7.0)
    part.rew_buf.fill_(3.0)
    ids = (torch.rand(n, generator=g) < 0.2).nonzero().flatten()
    env_list = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    env_list[:ids.numel()] = ids.to(DEV)
    count = torch.tensor([ids.numel()], dtype=torch.int32, device=DEV)
    kw = {"target_states": target} if kind == "strike" else {}
    part.observe_list(body, env_list, count, progress, **kw)
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids] = False
    obs = part.obs_buf.cpu()
    assert torch.equal(obs[ids], full.obs_buf.cpu()[ids])
    assert bool((obs[keep] == 7.0).all()) and bool((part.rew_buf == 3.0).all())
    assert int(part.reset_buf.abs().sum()) == 0 and int(part._terminate_buf.abs().sum()) == 0


def test_multinomial_with_replacement_does_not_synchronise():
    """The mixin draws clips with the reference's torch.multinomial (with replacement): it makes no host synchronisation, for one
    sample (a single env resetting) or many."""
    p = torch.rand(10, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        torch.multinomial(p, 1, replacement=True)
        torch.multinomial(p, 64, replacement=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)


@pytest.mark.parametrize("kind,upright,init", [("reach", True, "Random"), ("speed", False, "Random"), ("strike", True, "Random"),
                                               ("speed", True, "Start")])
def test_mixin_matches_oracle_with_the_reference_draws(env, kind, upright, init):
    """`HumanoidZTaskResetB200Mixin._reset_envs` on a stand-in task, seeded: the draws the reference's calls make in the reference's
    order, replayed into the oracle, give the same reset (the bars of test_reset_matches_oracle); the observation rows of the reset
    envs equal the full step kernel's; the gym setters get the reset envs' actor ids; a second reset makes no host synchronisation."""
    from pulse_b200.reach import ReachTaskB200
    from pulse_b200.ztask_reset import HumanoidZTaskResetB200Mixin
    from pulse_b200.ztasks import SpeedTaskB200, StrikeTaskB200
    from tests.ztask_standin import StandInZTask
    tb, ml, floor = env

    class Task(HumanoidZTaskResetB200Mixin, StandInZTask):
        pass

    n = 1024
    t = Task(kind, ml, DEV, n, state_init=init, upright=upright, seed=3)
    st = {"root_states": t._humanoid_root_states.cpu().clone(), "dof_pos": t._dof_pos.cpu().clone(), "dof_vel": t._dof_vel.cpu().clone(),
          "body_state": t._rigid_body_state_reshaped[:, :24].cpu().clone(), "sampled_motion_ids": t._sampled_motion_ids.cpu().clone(),
          "motion_start_times": t._motion_start_times.cpu().clone(), "progress_buf": t.progress_buf.cpu().clone(),
          "reset_buf": t.reset_buf.cpu().clone(), "terminate_buf": t._terminate_buf.cpu().clone(), "contact_forces": t._contact_forces.cpu().clone(),
          "amp_obs_buf": t._amp_obs_buf.cpu().clone(), "target_states": t._root_states[:, 1].cpu().clone()}
    obs0 = t.obs_buf.cpu().clone()
    st_pad = (t._dof_state[:, 69:].cpu().clone(), t._rigid_body_state_reshaped[:, 24:].cpu().clone())
    ids = (torch.rand(n, generator=torch.Generator().manual_seed(4)) < 0.1).nonzero().flatten()
    m = ids.numel()
    torch.manual_seed(77)
    t._reset_envs(ids.to(DEV))
    # the same calls, replayed
    torch.manual_seed(77)
    mids = torch.multinomial(ml._sampling_batch_prob, num_samples=m, replacement=True).cpu()
    ph = torch.rand(m, device=DEV).cpu() if init == "Random" else torch.zeros(m)
    su = torch.stack([torch.rand([m], device=DEV).cpu() for _ in range(4)], dim=1) if kind == "strike" else torch.zeros(m, 4)
    dr = {"motion_ids": torch.zeros(n, dtype=torch.int64), "phase": torch.zeros(n), "strike_u": torch.zeros(n, 4)}
    dr["motion_ids"][ids], dr["phase"][ids], dr["strike_u"][ids] = mids, ph, su
    exp = zo.ztask_reset(tb, st, ids, dr, floor, kind, upright=upright, state_init=zo.RANDOM if init == "Random" else zo.START, width=195)
    d = {"sampled_motion_ids": t._sampled_motion_ids, "motion_start_times": t._motion_start_times, "progress_buf": t.progress_buf,
         "reset_buf": t.reset_buf, "terminate_buf": t._terminate_buf, "amp_obs_buf": t._amp_obs_buf, "root_all": t._root_states,
         "dof_state": t._dof_state, "body": t._rigid_body_state_reshaped, "contact": t._contact_forces}
    _compare(d, exp, ids, n, kind, padding=False)
    assert torch.equal(t._dof_state[:, 69:].cpu(), st_pad[0]) and torch.equal(t._rigid_body_state_reshaped[:, 24:].cpu(), st_pad[1])
    if kind != "strike":
        tu = torch.rand([m, 3] if kind == "reach" else [m], device=DEV).cpu()
        lo, hi = 100, 200
        steps = torch.randint(low=lo, high=hi, size=(m,), device=DEV, dtype=torch.int64).cpu()
        if kind == "reach":
            want, wchg = zo.reach_task(tu, steps, torch.zeros(m, dtype=torch.int64), **zo.REACH)
            assert torch.equal(t._tar_pos.cpu()[ids], want) and torch.equal(t._tar_change_steps.cpu()[ids], wchg)
        else:
            want, wchg = zo.speed_task(tu, steps, torch.zeros(m, dtype=torch.int64), **zo.SPEED)
            assert torch.equal(t._tar_speed.cpu()[ids], want) and torch.equal(t._speed_change_steps.cpu()[ids], wchg)
            assert float(t.power_acc[ids.to(DEV)].abs().max()) == 0
    # observation rows of the reset envs = the full step kernel's on the state after the reset; the other rows untouched
    mk = {"reach": ReachTaskB200, "speed": SpeedTaskB200, "strike": StrikeTaskB200}[kind]
    ref = mk(n, device=DEV)
    if kind == "reach":
        ref._tar_pos = t._tar_pos
    if kind == "speed":
        ref._tar_speed = t._tar_speed
    if kind == "strike":
        ref.post_physics_step(t._rigid_body_state_reshaped, t.progress_buf, t._target_states, torch.zeros(n, 3, device=DEV))
    obs = t.obs_buf.cpu()
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids] = False
    assert torch.equal(obs[keep], obs0[keep])
    if kind == "strike":
        assert torch.equal(obs[ids], ref.obs_buf.cpu()[ids])
    else:
        # reach / speed: the observation precedes _reset_task (the reference's order), so only its self part is compared here
        assert torch.equal(obs[ids, :358], _self_obs_rows(t, ids, mk, n))
    assert [c[0] for c in t.gym_calls][:2] == ["set_actor_root_state_tensor_indexed", "set_dof_state_tensor_indexed"]
    assert torch.equal(t.gym_calls[0][1].cpu(), (2 * ids).int())
    # no host synchronisation in the mixin's own work once the floor table is built.  The reference's `_reset_env_tensors` clears its
    # counters with `buf[env_ids] = 0`, which copies the scalar from the host; that is the reference's code (the kernel has already
    # cleared them), so the check is suspended around it.
    ids2 = (torch.rand(n, generator=torch.Generator().manual_seed(5)) < 0.05).nonzero().flatten().to(DEV)
    reference_reset_env_tensors = t._reset_env_tensors

    def outside_the_check(env_ids):
        torch.cuda.set_sync_debug_mode(0)
        reference_reset_env_tensors(env_ids)
        torch.cuda.set_sync_debug_mode("error")

    t._reset_env_tensors = outside_the_check
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t._reset_envs(ids2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def _self_obs_rows(t, ids, mk, n):
    """The 358 self-observation columns the full step kernel writes for the state after the reset."""
    ref = mk(n, device=DEV)
    ref.post_physics_step(t._rigid_body_state_reshaped, t.progress_buf)
    return ref.obs_buf.cpu()[ids, :358]


def test_mixin_hands_default_and_hybrid_back_and_skips_empty_resets(env):
    from pulse_b200.ztask_reset import HumanoidZTaskResetB200Mixin
    from tests.ztask_standin import StandInZTask
    tb, ml, floor = env

    class Task(HumanoidZTaskResetB200Mixin, StandInZTask):
        pass

    for init in ("Default", "Hybrid"):
        with pytest.raises(AssertionError, match="reference reset path"):
            Task("reach", ml, DEV, 64, state_init=init)._reset_envs(torch.arange(3, device=DEV))
    t = Task("reach", ml, DEV, 64)
    before = t._rigid_body_state_reshaped.clone()
    t._reset_envs(torch.zeros(0, dtype=torch.int64, device=DEV))
    assert torch.equal(before, t._rigid_body_state_reshaped) and not t.gym_calls
