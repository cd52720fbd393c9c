"""Pedestrian terrain task on the device (pulse_terrain_step / pulse_traj_reset / pulse_terrain_heights) against the fixture written by the
unmodified reference (tests/golden/terrain.npz) and the oracle: reset / terminate bit-exact; height cells identical except points
within 1e-5 m of a cell boundary, which are listed; observations and rewards within 1e-4; trajectories from injected draws within
1e-5."""
import pytest
import torch

from oracle import terrain_oracle as to
from tests.test_terrain_cpu import CASES, CONTACT_IDS, DT, MAX_LEN, cell_heights, fixture, gen

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


BOUNDARY_M = 1e-5   # > the fp32 spacing of coordinates below 128 m (7.6e-6 m), where one rounding step can move a point across


def boundary_dist(points: torch.Tensor, hscale: float = 0.1) -> torch.Tensor:
    """[..., P] distance in metres from the point's x or y, whichever is nearer, to a cell boundary."""
    q = points[..., 0:2].double() / hscale
    return ((q - q.round()).abs() * hscale).min(dim=-1).values


def near_boundary(points: torch.Tensor) -> torch.Tensor:
    """[..., P] mask of the points listed as near a boundary: an fp32 rounding there may pick the neighbouring cell."""
    return boundary_dist(points) < BOUNDARY_M


def exempt(z, upright):
    """(per-point boundary distance of the head height map, per-env mask of rows whose center heights may pick another cell)."""
    bs = z["body_state"]
    grid = boundary_dist(to.grid_points_world(bs[:, to.HEAD_BODY_ID, 0:7], to.square_height_points(), upright))
    rows = near_boundary(to.center_points_world(bs[:, 0, 0:7], to.center_height_points(), upright)).any(dim=-1)
    rows |= near_boundary(to.center_points_world(z["root_states"][:, 0:7], to.center_height_points(), upright)).any(dim=-1)
    return grid, rows


def sim_views(z):
    from tests.terrain_standin import HumanoidPedestrianTerrainStandIn
    s = HumanoidPedestrianTerrainStandIn(z, DEV, z["heightfield"])
    return s._rigid_body_state_reshaped, s._humanoid_root_states, s._contact_forces, s.dof_force_tensor, s._dof_vel, s.progress_buf


def make_task(z, case, n=None, hf=True):
    from pulse_b200.terrain import PedestrianTerrainTaskB200, TerrainB200
    c = CASES[case]
    terrain = TerrainB200(z["heightfield"] if hf else None, device=DEV)
    t = PedestrianTerrainTaskB200(n or z["body_state"].shape[0], DEV, terrain, max_episode_length=MAX_LEN, dt=DT, upright=c["upright"],
                                  fuzzy_target=c["fuzzy"], power_reward=c["power"], use_center_height=c["use_center_height"])
    t.traj_verts.copy_(z["traj_verts"].to(DEV))
    return t


def check_obs(obs, want, grid, rows, tol=1e-4):
    obs, want = obs.cpu(), want.clone()
    keep = ~rows
    torch.testing.assert_close(obs[keep, :378], want[keep, :378], atol=tol, rtol=0)
    h, hw = obs[keep, 378:], want[keep, 378:]
    close = (h - hw).abs() <= tol
    ok = close | (grid[keep] < BOUNDARY_M)
    assert bool(ok.all()), (f"{int((~ok).sum())} height observations off outside the listed boundary points; their boundary distances "
                            f"{grid[keep][~ok].tolist()[:20]} m")


@pytest.mark.parametrize("case", sorted(CASES))
def test_step_matches_reference(case):
    z = fixture(case)
    t = make_task(z, case)
    rb, roots, cf, df, dv, prog = sim_views(z)
    t.post_physics_step(rb, roots, prog, cf, df, dv)
    torch.cuda.synchronize()
    assert torch.equal(t.reset_buf.cpu(), z[f"{case}_reset"]) and torch.equal(t._terminate_buf.cpu(), z[f"{case}_terminate"])
    torch.testing.assert_close(t.rew_buf.cpu(), z[f"{case}_rew"], atol=1e-4, rtol=0)
    torch.testing.assert_close(t.reward_raw.cpu(), z[f"{case}_reward_raw"], atol=1e-4, rtol=0)
    grid, rows = exempt(z, CASES[case]["upright"])
    print(f"exempt: {int((grid < BOUNDARY_M).sum())} boundary points, {int(rows.sum())} rows with a boundary center point")
    assert int(rows.sum()) < 20
    check_obs(t.obs_buf, torch.cat([z[f"{case}_self_obs"], z[f"{case}_task_obs"]], dim=1), grid, rows)


def test_heights_match_reference_cells():
    z = fixture()
    t = make_task(z, "a")
    bs = z["body_state"].to(DEV)
    h = t.get_heights(bs[:, to.HEAD_BODY_ID, 0:7].contiguous()).cpu()
    grid = exempt(z, True)[0] < BOUNDARY_M
    same = h == cell_heights(z)
    assert bool((same | grid).all()), f"{int((~(same | grid)).sum())} heights from another cell outside the boundary list"
    assert int(grid.sum()) < h.numel() // 100
    c = t.get_center_heights(bs[:, 0, 0:7].contiguous()).cpu()
    cmask = near_boundary(to.center_points_world(z["body_state"][:, 0, 0:7], to.center_height_points(), True))
    assert bool(((c == z["a_center_heights"]) | cmask).all())
    assert bool((t.get_center_heights(z["root_states"][:, 0:7].to(DEV).contiguous()).cpu() == z["a_root_center_heights"])
                .logical_or(near_boundary(to.center_points_world(z["root_states"][:, 0:7], to.center_height_points(), True))).all())


def test_traj_reset_matches_reference():
    z = fixture()
    draws, init = gen().reset_draws()
    nr = draws.shape[0]
    t = make_task(z, "a")
    t.traj_verts.zero_()
    t.reset_task(torch.arange(nr, device=DEV), init.to(DEV), rand=draws.to(DEV).contiguous())
    torch.cuda.synchronize()
    torch.testing.assert_close(t.traj_verts[:nr].cpu(), z["traj_reset_verts"], atol=1e-5, rtol=0)
    # Philox draws: same structure (start at the root, segment lengths within speed_max * dt), reproducible, fresh per call
    n = t.num_envs
    sel = [3, 7, 11]
    ids = torch.tensor(sel, device=DEV)
    v0 = t.traj_verts.clone()
    t.reset_task(ids, init[sel].to(DEV))
    v = t.traj_verts.cpu()
    assert torch.equal(v[sel, 0, 0:2], init[sel, 0:2])
    seg = (v[sel, 1:, 0:2] - v[sel, :-1, 0:2]).norm(dim=-1)
    assert float(seg.max()) <= 3.0 * t.traj_dt + 1e-4 and float(seg.mean()) > 0.01
    untouched = torch.ones(n, dtype=torch.bool)
    untouched[sel] = False
    assert torch.equal(v[untouched], v0.cpu()[untouched])
    first = v[sel].clone()
    t.reset_task(ids, init[sel].to(DEV))
    assert not torch.equal(t.traj_verts.cpu()[sel], first)


def test_env_ids_subset_equals_full():
    z = fixture()
    t = make_task(z, "a")
    rb, roots, cf, df, dv, prog = sim_views(z)
    t.compute_observations(rb, roots, prog)
    full = t.obs_buf.clone()
    t.obs_buf.fill_(-7.0)
    ids = torch.tensor([0, 5, 17, 100, 256], device=DEV)
    t.compute_observations(rb, roots, prog, env_ids=ids)
    assert torch.equal(t.obs_buf[ids], full[ids])
    others = torch.ones(t.num_envs, dtype=torch.bool, device=DEV)
    others[ids] = False
    assert bool((t.obs_buf[others] == -7.0).all())


def test_graph_replay_equals_eager():
    z = fixture("b")
    t = make_task(z, "b")
    rb, roots, cf, df, dv, prog = sim_views(z)
    t.post_physics_step(rb, roots, prog, cf, df, dv)
    torch.cuda.synchronize()
    eager = [x.clone() for x in (t.obs_buf, t.rew_buf, t.reward_raw, t.reset_buf, t._terminate_buf)]
    for x in (t.obs_buf, t.rew_buf, t.reward_raw):
        x.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        t.post_physics_step(rb, roots, prog, cf, df, dv)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        t.post_physics_step(rb, roots, prog, cf, df, dv)
    for x in (t.obs_buf, t.rew_buf, t.reward_raw):
        x.zero_()
    t.reset_buf.fill_(9)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, (t.obs_buf, t.rew_buf, t.reward_raw, t.reset_buf, t._terminate_buf)):
        assert torch.equal(a, b)


def synthetic(n, seed=3):
    """A 16384-env state over the env_pulse_terrain-sized heightfield region, for the oracle comparison at scale."""
    g = torch.Generator().manual_seed(seed)
    hf = torch.randint(-100, 400, (600, 800), generator=g, dtype=torch.int16)
    bs = torch.zeros(n, 24, 13)
    root = torch.rand(n, 3, generator=g) * torch.tensor([64.0, 84.0, 0.5]) + torch.tensor([-2.0, -2.0, 0.8])
    bs[..., 0:3] = root[:, None] + torch.randn(n, 24, 3, generator=g) * 0.3
    bs[:, 0, 0:3] = root
    bs[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 24, 4, generator=g), dim=-1)
    bs[..., 7:13] = torch.randn(n, 24, 6, generator=g)
    draws = torch.rand(n, to.TRAJ_DRAWS, generator=g)
    verts = torch.zeros(n, to.TRAJ_VERTS, 3)
    to.traj_reset(verts, torch.arange(n), root + torch.randn(n, 3, generator=g), draws, to.traj_params(MAX_LEN, DT), 2.0, 0.0, 3.0, 2.0, 0.02)
    contact = torch.randn(n, 24, 3, generator=g) * 20
    return dict(heightfield=hf, body_state=bs, root_states=bs[:, 0].clone(), progress_buf=torch.randint(0, 310, (n,), generator=g),
                contact_forces=contact, dof_force=torch.randn(n, 69, generator=g) * 30, dof_vel=torch.randn(n, 69, generator=g), traj_verts=verts)


@pytest.mark.parametrize("plane", [False, True])
def test_16384_envs_match_oracle(plane):
    n = 16384
    z = synthetic(n)
    t = make_task(z, "a", n=n, hf=not plane)
    rb, roots, cf, df, dv, prog = sim_views(z)
    t.post_physics_step(rb, roots, prog, cf, df, dv)
    torch.cuda.synchronize()
    want = to.terrain_step(None if plane else z["heightfield"], 0.1, 0.005, z["body_state"], z["root_states"], z["progress_buf"], z["contact_forces"],
                           torch.tensor(CONTACT_IDS), z["dof_force"], z["dof_vel"], z["traj_verts"], dt=DT, traj_dt=to.traj_params(MAX_LEN, DT),
                           max_episode_length=MAX_LEN)
    assert torch.equal(t.reset_buf.cpu(), want["reset"]) and torch.equal(t._terminate_buf.cpu(), want["terminate"])
    torch.testing.assert_close(t.rew_buf.cpu(), want["rew"], atol=1e-4, rtol=0)
    torch.testing.assert_close(t.reward_raw.cpu(), want["reward_raw"], atol=1e-4, rtol=1e-5)
    grid, rows = exempt(z, True)
    if plane:
        grid, rows = torch.full_like(grid, 1.0), torch.zeros_like(rows)
        assert float(t.obs_buf[:, 378:].abs().max()) == 0.0
    check_obs(t.obs_buf, want["obs"], grid, rows)


@pytest.mark.parametrize("case", sorted(CASES))
def test_mixin_fills_buffers_like_explicit_api(case):
    from pulse_b200.terrain import HumanoidPedestrianTerrainB200Mixin
    from tests.terrain_standin import HumanoidPedestrianTerrainStandIn
    z = fixture(case)
    c = CASES[case]

    class Task(HumanoidPedestrianTerrainB200Mixin, HumanoidPedestrianTerrainStandIn):
        pass
    m = Task(z, DEV, z["heightfield"], **{k: v for k, v in c.items() if k != "n"})
    m._compute_reward(None)
    m._compute_reset()
    m._compute_observations()
    t = make_task(z, case)
    rb, roots, cf, df, dv, prog = sim_views(z)
    t.post_physics_step(rb, roots, prog, cf, df, dv)
    torch.cuda.synchronize()
    for name in ("obs_buf", "rew_buf", "reward_raw", "reset_buf", "_terminate_buf"):
        assert torch.equal(getattr(m, name), getattr(t, name)), name
    ids = torch.tensor([2, 9], device=DEV)
    assert torch.equal(m._compute_task_obs(ids), t.obs_buf[ids, 358:])
    assert torch.equal(m._compute_humanoid_obs(ids), t.obs_buf[ids, :358])
    m._reset_task(ids)
    assert torch.equal(m._traj_gen._verts[ids, 0, 0:2], m._humanoid_root_states[ids, 0:2])


@pytest.mark.parametrize("option", ["_divide_group", "_group_obs", "velocity_map", "real_mesh", "_has_shape_obs", "big_ankle"])
def test_mixin_refuses_unsupported_options(option):
    from pulse_b200._lib import PulseError
    from pulse_b200.terrain import HumanoidPedestrianTerrainB200Mixin
    from tests.terrain_standin import HumanoidPedestrianTerrainStandIn
    z = fixture()

    class Task(HumanoidPedestrianTerrainB200Mixin, HumanoidPedestrianTerrainStandIn):
        pass
    m = Task(z, DEV, z["heightfield"], **{option: True})
    with pytest.raises(PulseError, match=option.lstrip("_")):
        m._compute_reward(None)
