"""Reference-state reset of the pedestrian terrain task (`pulse_reset_terrain`, the list observation of `pulse_terrain_step` and
`pulse_traj_reset_list`, through `pulse_b200.terrain_reset.TerrainResetB200`) against the CPU oracle tests/terrain_reset_oracle.py,
which tests/test_terrain_reset_cpu.py pins to the unmodified reference.

Bars (those of test_gpu_ztask_reset.py): env / actor lists, counts, clips, start times, location indices, counters and the cleared
contact forces bit-exact; simulator tensors within 1e-5 (bodies also rtol 2e-5), dof positions and AMP rows within 1e-4; every env that
is not reset bit-identical.  The root height carries the mean center height: envs whose center points lie within 1e-5 m of a cell
boundary may take the neighbouring cell (as test_gpu_terrain.py allows) and are exempt from that one comparison."""
import numpy as np
import pytest
import torch

from oracle import terrain_oracle as to
from tests import terrain_reset_oracle as tro
from tests import ztask_reset_oracle as zo
from tests.helpers import exact_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIPS = 23


@pytest.fixture(scope="module")
def env():
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.terrain import TerrainB200
    from pulse_b200.ztask_reset import smpl_ground_table
    from tests.golden.make_golden_terrain import heightfield
    tb = exact_tables(CLIPS, seed=9, min_frames=4, spread=120)
    floor = smpl_ground_table(tb.motion_aa, zo.StandInParser(), torch.linspace(-1.0, 1.0, 10))
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames",
                                                                 "dt", "length_starts")}, device=DEV)
    prob = torch.rand(CLIPS, generator=torch.Generator().manual_seed(4))
    prob[[1, 5, 11]] = 0.0
    ml._sampling_batch_prob = (prob / prob.sum()).to(DEV)
    hf = torch.from_numpy(heightfield())
    cx, cy = tro.walkable_table(tro.walkable_field(*hf.shape), 0.1, 5)
    return dict(tb=tb, ml=ml, floor=floor, hf=hf, cx=cx, cy=cy, terrain=TerrainB200(hf, device=DEV))


def _make(e, upright=True):
    from pulse_b200.terrain_reset import TerrainResetB200
    return TerrainResetB200(e["ml"], e["floor"].to(DEV), e["terrain"], e["cx"], e["cy"], upright=upright)


def _task(e, n):
    from pulse_b200.terrain import PedestrianTerrainTaskB200
    return PedestrianTerrainTaskB200(n, device=DEV, terrain=e["terrain"], dt=zo.DT, seed=11)


def _state(n, seed):
    g = torch.Generator().manual_seed(seed)
    st = {"root_states": torch.randn(n, 13, generator=g), "dof_pos": torch.randn(n, 69, generator=g), "dof_vel": torch.randn(n, 69, generator=g),
          "body_state": torch.randn(n, 24, 13, generator=g), "sampled_motion_ids": torch.randint(0, CLIPS, (n,), generator=g),
          "motion_start_times": torch.rand(n, generator=g), "progress_buf": torch.randint(0, 300, (n,), generator=g),
          "reset_buf": torch.zeros(n, dtype=torch.int64), "terminate_buf": (torch.rand(n, generator=g) < 0.3).long(),
          "contact_forces": torch.randn(n, 26, 3, generator=g), "amp_obs_buf": torch.randn(n, 10, 196, generator=g)}
    st["root_states"][:, 3:7] /= st["root_states"][:, 3:7].norm(dim=-1, keepdim=True)
    st["body_state"][..., 3:7] /= st["body_state"][..., 3:7].norm(dim=-1, keepdim=True)
    d = {k: st[k].to(DEV).clone() for k in ("sampled_motion_ids", "motion_start_times", "progress_buf", "reset_buf", "terminate_buf", "amp_obs_buf")}
    d["root_all"] = torch.full((n, 2, 13), 5.0, device=DEV)
    d["root_all"][:, 0] = st["root_states"].to(DEV)
    d["dof_state"] = torch.full((n, 72, 2), 5.0, device=DEV)
    d["dof_state"][:, :69, 0], d["dof_state"][:, :69, 1] = st["dof_pos"].to(DEV), st["dof_vel"].to(DEV)
    d["body"] = torch.full((n, 26, 13), 5.0, device=DEV)
    d["body"][:, :24] = st["body_state"].to(DEV)
    d["contact"] = st["contact_forces"].to(DEV).clone()
    d["actor_ids"] = torch.arange(n, dtype=torch.int32, device=DEV) * 2
    return st, d


def _draws(n, seed, prob, num_locations):
    g = torch.Generator().manual_seed(seed)
    return {"motion_ids": torch.multinomial(prob.cpu(), n, replacement=True, generator=g), "phase": torch.rand(n, generator=g),
            "loc_ids": torch.randint(0, num_locations, (n,), generator=g), "traj": torch.rand(n, to.TRAJ_DRAWS, generator=g)}


def _reset(r, d, env_ids=None, draws=None, **kw):
    inj = {} if draws is None else {k: draws[k].to(DEV) for k in ("motion_ids", "phase", "loc_ids")}
    return r.reset_envs(root_states=d["root_all"][:, 0], dof_pos=d["dof_state"][:, :69, 0], dof_vel=d["dof_state"][:, :69, 1],
                        rigid_body_state=d["body"], progress_buf=d["progress_buf"], sampled_motion_ids=d["sampled_motion_ids"],
                        motion_start_times=d["motion_start_times"], reset_buf=None if env_ids is not None else d["reset_buf"], env_ids=env_ids,
                        terminate_buf=d["terminate_buf"], contact_forces=d["contact"], amp_obs_buf=d["amp_obs_buf"], actor_ids=d["actor_ids"],
                        **inj, **kw)


def _boundary_envs(exp, ids, upright):
    """Reset envs (positions in ids) with a rotated center point within 1e-5 m of a cell boundary.  The middle point (offset 0) is
    the spawn point itself, a cell corner that both sides compute exactly."""
    rs = exp["root_states"][ids]
    pts = to.center_height_points()
    w = to.center_points_world(rs[:, 0:7], pts, upright)[:, pts[:, 0:2].abs().sum(dim=-1) > 0, 0:2] / 0.1
    return ((w - w.round()).abs() * 0.1 < 1e-5).any(dim=-1).any(dim=-1)


def _compare(d, exp, ids, n, upright):
    close = lambda a, b, **k: torch.testing.assert_close(a.cpu(), b, **({"atol": 1e-5, "rtol": 0} | k))
    for k in ("sampled_motion_ids", "progress_buf", "reset_buf", "terminate_buf"):
        assert torch.equal(d[k].cpu(), exp[k]), k
    assert torch.equal(d["motion_start_times"].cpu(), exp["motion_start_times"])
    got = d["root_all"][:, 0].cpu().clone()
    edge = _boundary_envs(exp, ids, upright)
    got[ids[edge], 2] = exp["root_states"][ids[edge], 2]                    # the exempt root heights
    close(got, exp["root_states"])
    assert int(edge.sum()) <= max(1, ids.numel() // 2)
    close(d["dof_state"][:, :69, 0], exp["dof_pos"], atol=1e-4, rtol=1e-4)
    close(d["dof_state"][:, :69, 1], exp["dof_vel"])
    close(d["body"][:, :24], exp["body_state"], rtol=2e-5)
    close(d["amp_obs_buf"], exp["amp_obs_buf"], atol=1e-4)
    assert torch.equal(d["contact"].cpu()[ids], torch.zeros(ids.numel(), 26, 3))
    keep = torch.ones(n, dtype=torch.bool)
    keep[ids] = False
    assert float((d["dof_state"][:, 69:] - 5.0).abs().max()) == 0 and float((d["body"][:, 24:] - 5.0).abs().max()) == 0
    assert float((d["root_all"][:, 1] - 5.0).abs().max()) == 0
    for ours, ref in ((d["root_all"][:, 0], exp["root_states"]), (d["body"][:, :24], exp["body_state"]), (d["amp_obs_buf"], exp["amp_obs_buf"]),
                      (d["dof_state"][:, :69, 0], exp["dof_pos"]), (d["contact"], exp["contact_forces"])):
        assert torch.equal(ours.cpu()[keep], ref[keep])
    if ids.numel():   # the root is lifted by the center height, the rigid bodies are not
        lifted = exp["center_height"].abs() > 1e-3
        body_z, root_z = d["body"][ids, 0, 2].cpu(), d["root_all"][ids, 0, 2].cpu()
        torch.testing.assert_close(root_z[~edge] - body_z[~edge], exp["center_height"][~edge], atol=2e-5, rtol=0)
        assert bool(lifted.any()) or ids.numel() < 8


CASES = [(1, 1.0, "list", True), (300, 0.05, "mask", True), (300, 0.5, "list", False), (2051, 0.5, "mask", True), (2051, 1.0, "list", False),
         (16384, 0.05, "list", True), (16384, 0.05, "mask", False), (16384, 1.0, "mask", True)]


@pytest.mark.parametrize("n,frac,mode,upright", CASES)
def test_reset_matches_oracle(env, n, frac, mode, upright):
    r = _make(env, upright)
    st, d = _state(n, seed=n)
    ids = (torch.rand(n, generator=torch.Generator().manual_seed(7)) < frac).nonzero().flatten()
    if n > 1:
        ids = torch.unique(torch.cat([ids, torch.tensor([0, n - 1])]))
    dr = _draws(n, 8, env["ml"]._sampling_batch_prob, r.num_locations)
    if mode == "mask":
        d["reset_buf"][ids.to(DEV)] = 1
        st["reset_buf"][ids] = 1
        ws = _reset(r, d, draws=dr)
    else:
        ws = _reset(r, d, env_ids=ids.to(DEV), draws=dr)
    exp = tro.terrain_reset(env["tb"], {k: v[:, :24] if k == "contact_forces" else v for k, v in st.items()}, ids, dr, env["floor"], env["hf"],
                            env["cx"], env["cy"], upright=upright)
    exp["contact_forces"] = st["contact_forces"].clone()
    exp["contact_forces"][ids] = 0
    torch.cuda.synchronize()
    cnt = int(ws["count"].item())
    assert cnt == ids.numel() and torch.equal(ws["env_list"][:cnt].cpu(), ids) and torch.equal(ws["actor_list"][:cnt].cpu(), (2 * ids).int())
    assert torch.equal(ws["loc_ids"].cpu()[ids], dr["loc_ids"][ids])
    _compare(d, exp, ids, n, upright)


def test_reset_observation_and_trajectories(env):
    """The list observation of the reset envs equals those rows of a full observation (stale waypoints included); the list
    trajectory reset with injected draws equals pulse_traj_reset on the same ids and roots."""
    n = 2051
    r, task = _make(env), _task(env, n)
    st, d = _state(n, seed=3)
    task.traj_verts.copy_(torch.randn(n, to.TRAJ_VERTS, 3, generator=torch.Generator().manual_seed(2)).to(DEV) * 5 + 10)
    ids = torch.arange(0, n, 3)
    dr = _draws(n, 9, env["ml"]._sampling_batch_prob, r.num_locations)
    _reset(r, d, env_ids=ids.to(DEV), draws=dr)
    task.obs_buf.fill_(7.0)
    r.observe(task, d["body"], d["root_all"][:, 0], d["progress_buf"])
    full = _task(env, n)
    full.traj_verts.copy_(task.traj_verts)
    full.compute_observations(d["body"], d["root_all"][:, 0], d["progress_buf"])
    keep = torch.ones(n, dtype=torch.bool, device=DEV)
    keep[ids.to(DEV)] = False
    assert torch.equal(task.obs_buf[ids.to(DEV)], full.obs_buf[ids.to(DEV)])
    assert bool((task.obs_buf[keep] == 7.0).all())
    # trajectories: list kernel vs pulse_traj_reset over the same ids, injected draws, bit for bit
    ref = _task(env, n)
    ref.traj_verts.copy_(task.traj_verts)
    r.reset_task(task, d["root_all"][:, 0], rand=dr["traj"].to(DEV).contiguous())
    ref.reset_task(ids.to(DEV), d["root_all"][ids.to(DEV), 0, 0:3], rand=dr["traj"][ids].to(DEV).contiguous())
    assert torch.equal(task.traj_verts, ref.traj_verts)
    torch.testing.assert_close(task.traj_verts[ids.to(DEV), 0, 0:2].cpu(), d["root_all"][ids.to(DEV), 0, 0:2].cpu(), rtol=0, atol=0)
    want = tro.reset_task(ref.traj_verts.cpu(), ids, d["root_all"][:, 0].cpu(), dr["traj"])
    torch.testing.assert_close(task.traj_verts.cpu(), want, atol=1e-4, rtol=1e-5)


def test_graph_replay_equals_eager_and_no_host_sync(env):
    """Reset + observation + trajectories captured in one CUDA graph with Philox draws and a device-side offset equal the eager calls
    at the same offsets, replay after replay; an eager reset runs under sync-debug mode "error"."""
    n = 4096
    outs = []
    for mode in ("eager", "graph"):
        r, task = _make(env), _task(env, n)
        st, d = _state(n, seed=5)
        off = torch.zeros(1, dtype=torch.int64, device=DEV)
        d["reset_buf"][::5] = 1
        reset0 = d["reset_buf"].clone()

        def step():
            d["reset_buf"].copy_(reset0)
            _reset(r, d, seed=77, offset=3, offset_dev=off)
            r.observe(task, d["body"], d["root_all"][:, 0], d["progress_buf"])
            r.reset_task(task, d["root_all"][:, 0], seed=78, offset=0, offset_dev=off)
        snaps = []
        if mode == "eager":
            for k in range(3):
                off.fill_(k)
                step()
                snaps.append([t.clone() for t in (d["root_all"], d["body"], d["amp_obs_buf"], task.obs_buf, task.traj_verts, d["sampled_motion_ids"])])
        else:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                step()
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
            # back to the eager run's starting point: the warm-up reset left its waypoints, which the next observation would read
            st, d0 = _state(n, seed=5)
            for k_, v in d0.items():
                d[k_].copy_(v)
            task.traj_verts.zero_()
            task.obs_buf.zero_()
            for k in range(3):
                off.fill_(k)
                g.replay()
                snaps.append([t.clone() for t in (d["root_all"], d["body"], d["amp_obs_buf"], task.obs_buf, task.traj_verts, d["sampled_motion_ids"])])
        outs.append(snaps)
    for a, b in zip(*outs):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert not torch.equal(outs[0][0][4], outs[0][1][4])           # another offset, other waypoints
    r, task = _make(env), _task(env, n)
    st, d = _state(n, seed=6)
    ids = torch.arange(0, n, 7, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _reset(r, d, env_ids=ids, seed=1)
        r.observe(task, d["body"], d["root_all"][:, 0], d["progress_buf"])
        r.reset_task(task, d["root_all"][:, 0])
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_philox_draw_statistics(env):
    """Philox location indices are uniform over the walkable table (chi-square); two successive trajectory resets of one env draw
    uncorrelated waypoints."""
    from scipy import stats
    from pulse_b200.terrain_reset import TerrainResetB200
    n, L = 16384, 64
    r = TerrainResetB200(env["ml"], env["floor"].to(DEV), env["terrain"], env["cx"][:L], env["cy"][:L])
    task = _task(env, n)
    st, d = _state(n, seed=12)
    ws = _reset(r, d, env_ids=torch.arange(n, device=DEV), seed=99, offset=5)
    counts = torch.bincount(ws["loc_ids"].cpu(), minlength=L).double()
    chi = stats.chisquare(counts.numpy())
    assert chi.pvalue > 1e-3, chi
    headings = []
    for k in range(2):
        r.reset_task(task, d["root_all"][:, 0], seed=5, offset=k)
        seg = task.traj_verts[:, 1, 0:2] - task.traj_verts[:, 0, 0:2]
        headings.append(torch.atan2(seg[:, 1], seg[:, 0]).cpu().double())
    corr = float(np.corrcoef(headings[0].numpy(), headings[1].numpy())[0, 1])
    assert abs(corr) < 0.05, corr
    assert abs(float(headings[0].mean())) < 0.1


def test_mixin_matches_oracle_with_the_reference_draws(env):
    """The mixin on a stand-in draws the reference's numbers (seeded torch and np.random), matches the oracle, writes the observation
    and new waypoints of the reset envs, leaves the task's _sampled_motion_ids alone, does nothing for an empty set and hands
    Default state init back to the reference."""
    import types
    from oracle import pulse_oracle as po
    from pulse_b200.terrain import HumanoidPedestrianTerrainB200Mixin
    from pulse_b200.terrain_reset import HumanoidPedestrianTerrainResetB200Mixin
    from tests.ztask_standin import StandInZTask

    class Task(HumanoidPedestrianTerrainResetB200Mixin, HumanoidPedestrianTerrainB200Mixin, StandInZTask):
        pass
    n = 300
    t = Task("speed", env["ml"], DEV, n)
    t._amp_obs_buf = torch.zeros(n, 10, 196, device=DEV)
    t._amp_root_height_obs, t.big_ankle, t.real_mesh = True, False, False
    t.cfg = {"env": {"terrain": {"terrainType": "trimesh"}, "use_center_height": True}}
    t.terrain = types.SimpleNamespace(heightsamples=env["hf"], horizontal_scale=0.1, vertical_scale=0.005, coord_x_scale=env["cx"],
                                      coord_y_scale=env["cy"])
    t.terrain_obs, t.terrain_obs_type, t.terrain_obs_root = True, "square", "head"
    t.height_points = to.square_height_points().expand(n, -1, -1).to(DEV)
    t._contact_body_ids = torch.tensor([7, 3, 8, 4], device=DEV)
    t.max_episode_length, t._enable_early_termination, t._fail_dist = 300, True, 4.0
    t._num_traj_samples, t._traj_sample_timestep = 10, 0.5
    t._speed_min, t._speed_max, t._accel_max, t._sharp_turn_prob = 0.0, 3.0, 2.0, 0.02
    t.fuzzy_target, t.power_reward, t.power_coefficient = False, False, 0.0005
    t._traj_gen = types.SimpleNamespace(_verts=torch.zeros(n, to.TRAJ_VERTS, 3, device=DEV))
    t.obs_buf = torch.zeros(n, 1402, device=DEV)
    t.rew_buf, t.reward_raw = torch.zeros(n, device=DEV), torch.zeros(n, 2, device=DEV)
    t._reset_envs(torch.zeros(0, dtype=torch.int64, device=DEV))
    before = {k: v.clone() for k, v in (("rb", t._rigid_body_state_reshaped), ("root", t._root_states), ("amp", t._amp_obs_buf))}
    assert all(torch.equal(before[k], v) for k, v in (("rb", t._rigid_body_state_reshaped), ("root", t._root_states), ("amp", t._amp_obs_buf)))
    st = {"root_states": t._humanoid_root_states.cpu().clone(), "dof_pos": t._dof_pos.cpu().clone(), "dof_vel": t._dof_vel.cpu().clone(),
          "body_state": t._rigid_body_state_reshaped[:, :24].cpu().clone(), "sampled_motion_ids": torch.zeros(n, dtype=torch.int64),
          "motion_start_times": torch.zeros(n), "progress_buf": t.progress_buf.cpu().clone(), "reset_buf": t.reset_buf.cpu().clone(),
          "terminate_buf": t._terminate_buf.cpu().clone(), "contact_forces": t._contact_forces[:, :24].cpu().clone(), "amp_obs_buf": t._amp_obs_buf.cpu().clone()}
    sampled0 = t._sampled_motion_ids.clone()
    ids = torch.arange(0, n, 4, device=DEV)
    torch.manual_seed(21)
    np.random.seed(21)
    m = len(ids)
    dr = {"motion_ids": torch.zeros(n, dtype=torch.int64), "phase": torch.zeros(n), "loc_ids": torch.zeros(n, dtype=torch.int64)}
    dr["motion_ids"][ids.cpu()] = torch.multinomial(env["ml"]._sampling_batch_prob, num_samples=m, replacement=True).cpu()
    dr["phase"][ids.cpu()] = torch.rand(m, device=DEV).cpu()
    dr["loc_ids"][ids.cpu()] = torch.from_numpy(np.random.randint(0, env["cx"].shape[0], size=m).astype(np.int64))
    torch.manual_seed(21)
    np.random.seed(21)
    t._reset_envs(ids)
    exp = tro.terrain_reset(env["tb"], st, ids.cpu(), dr, env["floor"], env["hf"], env["cx"], env["cy"])
    torch.cuda.synchronize()
    edge = _boundary_envs(exp, ids.cpu(), True)
    got = t._humanoid_root_states.cpu().clone()
    got[ids.cpu()[edge], 2] = exp["root_states"][ids.cpu()[edge], 2]
    torch.testing.assert_close(got, exp["root_states"], atol=1e-5, rtol=0)
    torch.testing.assert_close(t._rigid_body_state_reshaped[:, :24].cpu(), exp["body_state"], atol=1e-5, rtol=2e-5)
    torch.testing.assert_close(t._amp_obs_buf.cpu(), exp["amp_obs_buf"], atol=1e-4, rtol=0)
    assert torch.equal(t._reset_ref_motion_ids.cpu(), dr["motion_ids"][ids.cpu()])
    assert torch.equal(t._sampled_motion_ids, sampled0)
    assert bool((t.obs_buf[ids].abs().sum(dim=-1) > 0).all()) and float(t.obs_buf[1::4].abs().max()) == 0
    torch.testing.assert_close(t._traj_gen._verts[ids, 0, 0:2], t._humanoid_root_states[ids, 0:2], atol=0, rtol=0)
    assert float(t._traj_gen._verts[1::4].abs().max()) == 0
    t._state_init = types.SimpleNamespace(name="Hybrid")
    with pytest.raises(AssertionError, match="reference reset path"):
        t._reset_envs(ids)
