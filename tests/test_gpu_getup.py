"""Getup reset (`pulse_reset_getup` / `pulse_getup_amp_init`) against the oracle of tests/getup_oracle.py, which the CPU suite pins to
the reference's `HumanoidImGetup._reset_actors` (tests/golden/getup.npz).

Bars: lists, counts, classes, assignments, availability, counters and the fall-pool copies bit-exact; the reference-state envs within
test_gpu_reset's tolerances; every env that is not reset, and every buffer a class does not write, bit-identical."""
import pytest
import torch

from tests import getup_oracle as go
from tests.test_gpu_reset import DEV, _device_state, _setup

pytestmark = pytest.mark.gpu


def _getup_state(n, seed, term_frac, pool=None):
    po, tb, comp, st, g = _setup(n, seed=seed)
    P = pool or n
    st["terminate_buf"] = (torch.rand(n, generator=g) < term_frac).long()
    st["recovery_counter"] = torch.randint(0, 5, (n,), generator=g, dtype=torch.int32)
    st["avail"] = (torch.rand(P, generator=g) < 0.3).long()
    st["fid"] = torch.randint(0, P, (n,), generator=g)        # arbitrary, often stale: the release frees whatever they point at
    st["fall_root"], st["fall_dof_pos"], st["fall_dof_vel"] = torch.randn(P, 13, generator=g), torch.randn(P, 69, generator=g), torch.randn(P, 69, generator=g)
    return po, tb, comp, st, g


def _device(st, n):
    d = _device_state(st, n)
    d["fall_dof"] = torch.stack([st["fall_dof_pos"], st["fall_dof_vel"]], -1).to(DEV)     # [P, 69, 2]: strided views like the dof state
    return d


def _call(comp, d, p_rec, p_fall, steps=60, env_ids=None, draws=None, **kw):
    rec_u, fall_u, keys = (None, None, None) if draws is None else (x.to(DEV) for x in draws)
    return comp.reset_getup(motion_ids=d["motion_ids"], motion_start_times=d["start_times"], motion_start_offset=d["start_offset"],
                            global_offset=d["global_offset"], progress_buf=d["progress_buf"], root_states=d["root_all"][:, 0],
                            dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1], rigid_body_state=d["body"],
                            reset_buf=None if env_ids is not None else d["reset_buf"], env_ids=env_ids, terminate_buf=d["terminate_buf"],
                            cycle_counter=d["cycle_counter"], contact_forces=d["contact"], amp_obs_buf=d["amp_obs_buf"], actor_ids=d["actor_ids"],
                            recovery_counter=d["recovery_counter"], available_fall_states=d["avail"], fall_id_assignments=d["fid"],
                            fall_root_states=d["fall_root"], fall_dof_pos=d["fall_dof"][..., 0], fall_dof_vel=d["fall_dof"][..., 1],
                            recovery_prob=p_rec, fall_prob=p_fall, recovery_steps=steps, recovery_u=rec_u, fall_u=fall_u, fall_keys=keys, **kw)


def _check(d, ws, exp, info, ids, n):
    torch.cuda.synchronize()
    cnt = int(ws["count"].item())
    assert cnt == ids.numel() and torch.equal(ws["env_list"][:cnt].cpu(), ids) and torch.equal(ws["actor_list"][:cnt].cpu(), (ids * 2).int())
    cc = ws["class_counts"].cpu().tolist()
    assert cc == [info["ref_ids"].numel(), info["fall_ids"].numel(), info["recovery_ids"].numel()]
    for key, k in (("ref_list", "ref_ids"), ("fall_list", "fall_ids"), ("recovery_list", "recovery_ids")):
        assert torch.equal(ws[key][:info[k].numel()].cpu(), info[k]), key
    assert torch.equal(ws["env_class"].cpu()[ids], info["classes"][ids])
    assert torch.equal(ws["fall_pick"][:cc[1]].cpu(), info["fall_states"])
    for k in ("progress_buf", "reset_buf", "terminate_buf", "cycle_counter", "recovery_counter", "avail", "fid", "start_times", "start_offset",
              "global_offset"):
        assert torch.equal(d[k].cpu(), exp[k]), k
    ref = torch.zeros(n, dtype=torch.bool)
    ref[info["ref_ids"]] = True
    exact = lambda a, b: torch.equal(a.cpu()[~ref], b[~ref])
    close = lambda a, b, **k: torch.testing.assert_close(a.cpu(), b, **({"atol": 1e-4, "rtol": 0} | k))
    for ours, theirs, tol in ((d["root_all"][:, 0], exp["root_states"], dict(atol=1e-5)), (d["dof_state"][:, :69, 0], exp["dof_pos"], dict(rtol=1e-4)),
                              (d["dof_state"][:, :69, 1], exp["dof_vel"], dict(atol=1e-5)), (d["body"][:, :24], exp["body_state"], dict(atol=1e-5, rtol=2e-5)),
                              (d["amp_obs_buf"], exp["amp_obs_buf"], {})):
        # fall-pool copies and untouched envs: bit for bit.  The reference-state rows: test_gpu_reset's bars; at 16384 envs a few of the
        # slerped body rotations (4 of 5.1 M floats) land 1.06e-5 from the oracle, hence the relative term on the bodies
        assert exact(ours, theirs)
        close(ours, theirs, **tol)
    close(d["contact"][:, :24], exp["contact_forces"], atol=0)
    assert float(d["contact"][ids].abs().max() if ids.numel() else 0) == 0
    assert float((d["root_all"][:, 1] - 5.0).abs().max()) == 0 and float((d["dof_state"][:, 69:] - 5.0).abs().max()) == 0


CASES = [  # n, mode, reset fraction, terminate fraction, recovery_prob, fall_prob
    (300, "mask", 0.4, 0.3, 0.5, 0.5),
    (300, "list", 0.0, 0.3, 0.5, 0.5),          # empty reset set
    (300, "mask", 1.0, 1.0, 1.0, 0.0),          # full set, every env recovers
    (2051, "list", 1.0, 0.0, 1.0, 1.0),         # nobody terminated: every env falls
    (2051, "mask", 0.13, 0.3, 0.0, 1.0),
    (2051, "list", 0.5, 1.0, 0.3, 0.0),
    (16384, "mask", 0.05, 0.3, 0.3, 0.1),       # env_im_vae.yaml's probabilities
    (16384, "list", 0.5, 0.3, 0.3, 0.1),
]


@pytest.mark.parametrize("n,mode,frac,term,p_rec,p_fall", CASES)
def test_reset_getup_matches_oracle(n, mode, frac, term, p_rec, p_fall):
    po, tb, comp, st, g = _getup_state(n, seed=n % 97, term_frac=term)
    mask = torch.rand(n, generator=g) < frac
    ids = mask.nonzero().flatten()
    st["reset_buf"] = mask.long() * 3 if mode == "mask" else torch.zeros(n, dtype=torch.long)   # a list call has no mask to clear
    phase, draws = torch.rand(n, generator=g), (torch.rand(n, generator=g), torch.rand(n, generator=g), torch.rand(n, generator=g))
    d = _device(st, n)
    ws = _call(comp, d, p_rec, p_fall, env_ids=ids.to(DEV) if mode == "list" else None, draws=draws, phase=phase.to(DEV))
    exp, info = go.getup_reset(tb, po.ImStepConfig(), st, ids, phase, *draws, p_rec, p_fall, 60)
    _check(d, ws, exp, info, ids, n)
    assert int(ws["error"].item()) == info["shortfall"]       # held states nobody is assigned to can outnumber the free ones


def test_stale_release_frees_a_state_another_env_holds():
    """humanoid_im_getup.py:136: env 0's stale assignment points at the state env 1 holds; resetting env 0 (a reference-state episode)
    frees it, so the next fall env takes it while env 1 still has it assigned."""
    n = 64
    po, tb, comp, st, g = _getup_state(n, seed=4, term_frac=0.0)
    st["avail"].zero_()
    st["fid"].zero_()
    st["avail"][5], st["fid"][0], st["fid"][1] = 1, 5, 5
    ids = torch.tensor([0, 7])
    phase, rec_u = torch.rand(n, generator=g), torch.ones(n)
    fall_u = torch.ones(n)
    fall_u[7] = 0.0
    keys = torch.ones(n)
    keys[5] = 0.0                                          # state 5 has the smallest key: env 7 gets it
    d = _device(st, n)
    ws = _call(comp, d, 0.5, 0.5, env_ids=ids.to(DEV), draws=(rec_u, fall_u, keys), phase=phase.to(DEV))
    exp, info = go.getup_reset(tb, po.ImStepConfig(), st, ids, phase, rec_u, fall_u, keys, 0.5, 0.5, 60)
    _check(d, ws, exp, info, ids, n)
    assert d["fid"][7].item() == 5 and d["fid"][1].item() == 5 and d["avail"][5].item() == 1


def test_exhausted_pool_gives_surplus_a_reference_state_episode():
    n, P = 300, 20
    po, tb, comp, st, g = _getup_state(n, seed=5, term_frac=0.0, pool=P)
    st["avail"].zero_()
    st["avail"][:8] = 1
    st["fid"] = torch.randint(8, P, (n,), generator=g)
    ids = torch.arange(0, n, 5)
    phase, draws = torch.rand(n, generator=g), (torch.ones(n), torch.zeros(n), torch.rand(P, generator=g))
    d = _device(st, n)
    ws = _call(comp, d, 0.3, 1.0, env_ids=ids.to(DEV), draws=draws, phase=phase.to(DEV))
    exp, info = go.getup_reset(tb, po.ImStepConfig(), st, ids, phase, *draws, 0.3, 1.0, 60)
    assert info["shortfall"] > 0
    _check(d, ws, exp, info, ids, n)
    assert int(ws["error"].item()) == info["shortfall"]
    with pytest.raises(Exception, match="no free fall state"):
        comp.check_getup_error()


def test_reset_getup_philox_draws():
    """Without injected draws: recovery share among the terminated envs and fall share among the rest within 5 sigma of p, the fall
    states of one call distinct and free, and the same (seed, offset) reproducing every output."""
    n, p_rec, p_fall = 16384, 0.3, 0.2
    po, tb, comp, st, g = _getup_state(n, seed=21, term_frac=0.5)
    st["reset_buf"] = torch.ones(n, dtype=torch.long)
    free = st["avail"].clone()
    free[st["fid"]] = 0
    runs = []
    for _ in range(2):
        d = _device(st, n)
        ws = _call(comp, d, p_rec, p_fall, seed=77, offset=5)
        torch.cuda.synchronize()
        runs.append(({k: v.clone() for k, v in d.items()}, {k: v.clone() for k, v in ws.items()}))
    (d, ws), (d2, ws2) = runs
    for k in d:
        assert torch.equal(d[k], d2[k]), k
    for k in ws:
        assert torch.equal(ws[k], ws2[k]), k
    cls = ws["env_class"].cpu()
    term = st["terminate_buf"] == 1
    n_t, n_rest = int(term.sum()), int((~(cls == go.RECOVERY)).sum())
    rec_share = float((cls[term] == go.RECOVERY).float().mean())
    assert abs(rec_share - p_rec) < 5 * (p_rec * (1 - p_rec) / n_t) ** 0.5
    fall_share = float((cls[cls != go.RECOVERY] == go.FALL).float().mean())
    assert abs(fall_share - p_fall) < 5 * (p_fall * (1 - p_fall) / n_rest) ** 0.5
    k = int(ws["class_counts"][1])
    picks = ws["fall_pick"][:k].cpu()
    assert picks.unique().numel() == k and bool((free[picks] == 0).all())
    assert torch.equal(d["fid"].cpu()[ws["fall_list"][:k].cpu()], picks)


def test_reset_getup_in_a_cuda_graph():
    """Captured once, replayed with the device-side offset advancing: each replay equals an eager call at the same offset."""
    n = 2051
    po, tb, comp, st, g = _getup_state(n, seed=31, term_frac=0.4)
    st["reset_buf"] = (torch.rand(n, generator=g) < 0.2).long()
    d = _device(st, n)
    init = {k: v.clone() for k, v in d.items()}
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    restore = lambda: [d[k].copy_(v) for k, v in init.items()]
    _call(comp, d, 0.4, 0.3, seed=9, offset_dev=off)       # allocates the workspace
    torch.cuda.synchronize()
    graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        restore()
        with torch.cuda.graph(graph, stream=s):
            ws = _call(comp, d, 0.4, 0.3, seed=9, offset_dev=off)
    torch.cuda.current_stream().wait_stream(s)
    for step in (3, 4, 11):
        restore()
        off.fill_(step)
        graph.replay()
        torch.cuda.synchronize()
        got = ({k: v.clone() for k, v in d.items()}, {k: v.clone() for k, v in ws.items()})
        restore()
        ws_e = _call(comp, d, 0.4, 0.3, seed=9, offset_dev=off)
        torch.cuda.synchronize()
        for k in d:
            assert torch.equal(got[0][k], d[k]), (step, k)
        for k in ("count", "class_counts", "env_class", "env_list"):
            assert torch.equal(got[1][k], ws_e[k]), (step, k)
    assert int(got[1]["class_counts"][1]) > 0 and int(got[1]["class_counts"][2]) > 0


def test_getup_amp_init_matches_oracle():
    n = 2051
    po, tb, comp, st, g = _getup_state(n, seed=41, term_frac=0.5)
    mask = torch.rand(n, generator=g) < 0.3
    ids = mask.nonzero().flatten()
    st["reset_buf"] = mask.long()
    phase, draws = torch.rand(n, generator=g), (torch.rand(n, generator=g), torch.rand(n, generator=g), torch.rand(n, generator=g))
    d = _device(st, n)
    _call(comp, d, 0.5, 0.5, draws=draws, phase=phase.to(DEV))
    exp, info = go.getup_reset(tb, po.ImStepConfig(), st, ids, phase, *draws, 0.5, 0.5, 60)
    body = torch.randn(n, 26, 13, generator=g)              # the simulator state after its refresh
    body[..., 3:7] = torch.nn.functional.normalize(body[..., 3:7], dim=-1)
    d["body"].copy_(body.to(DEV))
    amp0 = d["amp_obs_buf"].cpu()
    comp.getup_amp_init(body_state=d["body"], dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1], amp_obs_buf=d["amp_obs_buf"])
    torch.cuda.synchronize()
    want = go.getup_amp_init(amp0, body[:, :24], d["dof_state"][:, :69, 0].cpu(), d["dof_state"][:, :69, 1].cpu(), info["fall_ids"],
                             info["recovery_ids"])
    assert info["fall_ids"].numel() > 0 and info["recovery_ids"].numel() > 0
    torch.testing.assert_close(d["amp_obs_buf"].cpu(), want, atol=1e-4, rtol=0)
    touched = torch.zeros(n, dtype=torch.bool)
    touched[torch.cat([info["fall_ids"], info["recovery_ids"]])] = True
    assert torch.equal(d["amp_obs_buf"].cpu()[~touched], amp0[~touched])
    assert torch.equal(d["amp_obs_buf"].cpu()[info["recovery_ids"], 1:], amp0[info["recovery_ids"], 1:])


def test_getup_mixin_reset_envs_without_host_sync():
    """HumanoidImGetupB200Mixin._reset_envs on a getup stand-in: the oracle composite for the same torch.rand draws, after the
    stand-in's refresh (the simulator's rigid bodies, restored for the reference-state envs only), under sync-debug mode "error"."""
    from pulse_b200.humanoid_im import HumanoidImGetupB200Mixin
    from tests.helpers import exact_step_inputs, exact_tables
    from tests.standins import StandInHumanoidIm
    from tests.test_gpu_boundary import _mlib

    class GetupStandIn(StandInHumanoidIm):
        """HumanoidImGetup's reset state (humanoid_im_getup.py:44-62, :92-123) on top of the HumanoidIm stand-in."""

        def __init__(self, motion_lib, z, device, pool_seed=0):
            super().__init__(motion_lib, z, device, getup=True)
            n, g = self.num_envs, torch.Generator().manual_seed(pool_seed)
            self._recovery_episode_prob, self._fall_init_prob, self._recovery_steps = 0.5, 0.4, 60
            self.availalbe_fall_states = torch.zeros(n, dtype=torch.long, device=device)
            self.fall_id_assignments = torch.zeros(n, dtype=torch.long, device=device)
            self._fall_root_states = torch.randn(n, 13, generator=g).to(device)
            self._fall_dof_pos, self._fall_dof_vel = torch.randn(n, 69, generator=g).to(device), torch.zeros(n, 69, device=device)
            self._reset_fall_env_ids = []

        def _reset_env_tensors(self, env_ids):
            # the stand-in's humanoid.py:589-609 with index_fill_: `x[ids] = 0` copies its scalar from host memory, which the sync
            # check below would report although no simulator tensor needs it
            env_ids_int32 = self._humanoid_actor_ids[env_ids]
            self.gym_calls.append(("set_actor_root_state_tensor_indexed", env_ids_int32.clone(), len(env_ids_int32)))
            self.gym_calls.append(("set_dof_state_tensor_indexed", env_ids_int32.clone(), len(env_ids_int32)))
            for t in (self.progress_buf, self.reset_buf, self._terminate_buf, self._contact_forces):
                t.index_fill_(0, env_ids, 0)

    class Task(HumanoidImGetupB200Mixin, GetupStandIn):
        pass

    from oracle import pulse_oracle as po
    n = 389
    tb = exact_tables(41, seed=8)
    z, _ = exact_step_inputs(tb, n, seed=9)
    task = Task(_mlib(tb), z, DEV)
    task._terminate_buf.copy_((torch.arange(n, device=DEV) % 3 == 0).long())
    task._pulse_setup()
    amp0 = torch.randn(n, 10, 196, device=DEV)
    task._amp_obs_buf.copy_(amp0)
    ids = torch.arange(0, n, 2, device=DEV)
    snap = {k: getattr(task, a).clone().cpu() for k, a in (("avail", "availalbe_fall_states"), ("fid", "fall_id_assignments"),
                                                          ("recovery_counter", "_recovery_counter"), ("terminate_buf", "_terminate_buf"))}
    sim_body = task._sim_rigid_body_state.cpu()
    torch.manual_seed(123)
    torch.cuda.set_sync_debug_mode("error")
    try:
        task._reset_envs(ids)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    torch.manual_seed(123)
    phase = torch.zeros(n, device=DEV)
    phase[ids] = torch.rand(ids.shape, device=DEV)
    u = torch.ones(2, n, device=DEV)
    u[:, ids] = torch.rand((2, ids.numel()), device=DEV)
    keys = torch.rand(n, device=DEV)
    st = {"motion_ids": z["motion_ids"], "start_times": z["start_times"], "start_offset": z["start_offset"], "global_offset": z["global_offset"],
          "cycle_counter": z["cycle_counter"], "progress_buf": z["progress_buf"] - 1, "reset_buf": torch.ones(n, dtype=torch.long),
          "root_states": torch.zeros(n, 13), "dof_pos": z["dof_pos"], "dof_vel": z["dof_vel"], "body_state": z["body_state"],
          "contact_forces": torch.ones(n, 24, 3), "amp_obs_buf": amp0.cpu(), "obs_buf": torch.zeros(n, 934), "dof_force": z["dof_force"],
          "fall_root": task._fall_root_states.cpu(), "fall_dof_pos": task._fall_dof_pos.cpu(), "fall_dof_vel": task._fall_dof_vel.cpu(), **snap}
    exp, info = go.getup_reset(tb, po.ImStepConfig(), st, ids.cpu(), phase.cpu(), u[0].cpu(), u[1].cpu(), keys.cpu(), 0.5, 0.4, 60)
    assert info["fall_ids"].numel() > 0 and info["recovery_ids"].numel() > 0 and info["ref_ids"].numel() > 0
    for k, a in (("avail", "availalbe_fall_states"), ("fid", "fall_id_assignments"), ("recovery_counter", "_recovery_counter"),
                 ("progress_buf", "progress_buf"), ("terminate_buf", "_terminate_buf"), ("start_times", "_motion_start_times")):
        assert torch.equal(getattr(task, a).cpu(), exp[k]), k
    torch.testing.assert_close(task._humanoid_root_states.cpu(), exp["root_states"], atol=1e-5, rtol=0)
    torch.testing.assert_close(task._dof_pos.cpu(), exp["dof_pos"], atol=1e-4, rtol=1e-4)
    # after the refresh: the reference pose where a reference-state episode began, the simulator's bodies everywhere else
    body = sim_body.clone()
    body[info["ref_ids"], :24] = exp["body_state"][info["ref_ids"]]
    torch.testing.assert_close(task._rigid_body_state_reshaped.cpu(), body, atol=1e-5, rtol=0)
    want = go.getup_amp_init(exp["amp_obs_buf"], body[:, :24], task._dof_pos.cpu(), task._dof_vel.cpu(), info["fall_ids"], info["recovery_ids"])
    torch.testing.assert_close(task._amp_obs_buf.cpu(), want, atol=1e-4, rtol=0)
    assert len(task.gym_calls) == 2 and torch.equal(task.gym_calls[0][1].cpu(), (ids.cpu() * 2).int())
