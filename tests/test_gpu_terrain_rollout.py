"""The pedestrian terrain task's rollout on the device (`pulse_b200.terrain_rollout.TerrainStepsB200`), the rollout side of `SeptPolicy`
and `pulse_terrain_rollout_step`.

Bars: the sept rollout entry points bit for bit against `act()` and against each other (the sampling at the bar of test_gpu_rollout.py);
the rollout step bit for bit against advancing the counter and `pulse_terrain_step(STEP_ALL)`; the driver over two separate uploads of
one map bit for bit against the driver over one; the Philox blocks `philox_blocks` names, regenerated on the host and injected,
against the kernels' own draws; three eager driver steps, with resets,
bit for bit against the same steps composed from the existing public calls; the graph-captured, stream-overlapped horizon against the
sequential eager one bit for bit over eager, capture and replay; hook mode against the sequential order; `finish` and `train_epoch`
against the same calls issued separately; a replayed iteration without host synchronisation.  Fixtures are seeded synthetic state over
a small synthetic heightfield with steps and slopes; every case runs once."""
import pytest
import torch

from tests import terrain_reset_oracle as tro
from tests.helpers import exact_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIPS = 23


@pytest.fixture(scope="module")
def env():
    from pulse_b200.motion_lib import MotionLibB200
    from pulse_b200.terrain import TerrainB200
    from tests.golden.make_golden_terrain import heightfield
    tb = exact_tables(CLIPS, seed=9, min_frames=4, spread=120)
    ml = MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames",
                                                                 "dt", "length_starts")}, device=DEV)
    g = torch.Generator().manual_seed(2)
    floor = (-0.9 + 0.05 * torch.rand(tb.motion_aa.shape[0], generator=g)).to(DEV)
    hf = torch.from_numpy(heightfield())
    cx, cy = tro.walkable_table(tro.walkable_field(*hf.shape), 0.1, 5)
    return dict(ml=ml, floor=floor, hf=hf, cx=cx, cy=cy, terrain=TerrainB200(hf, device=DEV))


def _sim(n, seed, extent):
    """Isaac-Gym shaped simulator tensors (2 actors per env, 72 dofs x (pos, vel), 26 bodies) over the heightfield.  Every 7th env
    carries a contact force on a non-contact body (early termination), every 11th is at the end of its episode, the others are early
    in theirs."""
    g = torch.Generator().manual_seed(seed)
    root_xy = torch.rand(n, 2, generator=g) * (torch.tensor(extent) - 4.0) + 2.0
    body = torch.zeros(n, 26, 13)
    body[..., 0:2] = root_xy[:, None] + 0.2 * torch.randn(n, 26, 2, generator=g)
    body[..., 2] = 0.9 + 0.3 * torch.randn(n, 26, generator=g)
    body[..., 3:7] = torch.nn.functional.normalize(torch.randn(n, 26, 4, generator=g), dim=-1)
    body[..., 7:13] = torch.randn(n, 26, 6, generator=g)
    contact = torch.zeros(n, 26, 3)
    contact[::7, 5, 2] = 60.0
    progress = torch.randint(0, 20, (n,), generator=g)
    progress[::7] = progress[::7].clamp(min=2)                  # the contact test needs progress > 1
    progress[::11] = 298
    root = torch.zeros(n, 2, 13)
    root[:, 0] = body[:, 0]
    root[:, 1, 6] = 1.0
    sim = dict(body_state=body, root_all=root, dof_state=torch.randn(n, 72, 2, generator=g), contact_forces=contact, progress_buf=progress,
               sampled_motion_ids=torch.randint(0, CLIPS, (n,), generator=g), motion_start_times=torch.rand(n, generator=g),
               dof_force=torch.randn(n, 69, generator=g), actor_ids=torch.arange(n, dtype=torch.int32) * 2)
    sim = {k: v.to(DEV) for k, v in sim.items()}
    sim.update(root_states=sim["root_all"][:, 0], dof_pos=sim["dof_state"][:, :69, 0], dof_vel=sim["dof_state"][:, :69, 1])
    return sim


def _policy(seed=0):
    from pulse_b200.sept import SeptPolicy
    pol = SeptPolicy(num_actions=32, with_disc=False, device=DEV, seed=seed)
    g = torch.Generator().manual_seed(seed + 40)
    pol.obs_rms.running_mean.copy_(0.1 * torch.randn(pol.obs_size, generator=g, dtype=torch.float64))
    pol.obs_rms.running_var.copy_(0.5 + torch.rand(pol.obs_size, generator=g, dtype=torch.float64))
    pol.obs_rms._refresh()
    pol.value_rms.running_mean.fill_(0.7)
    pol.value_rms.running_var.fill_(2.3)
    pol.value_rms._refresh()
    return pol


def _driver(env, n, T=4, seed=5, use_graphs=True, power=False, task_terrain=None, reset=None):
    """`task_terrain` / `reset`: the task's heightfield and the reset, by default both over the fixture's one TerrainB200."""
    from pulse_b200.terrain import PedestrianTerrainTaskB200
    from pulse_b200.terrain_reset import TerrainResetB200
    from pulse_b200.terrain_rollout import TerrainStepsB200
    from pulse_b200.vae import PulseVAE
    task = PedestrianTerrainTaskB200(n, device=DEV, terrain=task_terrain or env["terrain"], power_reward=power, seed=11)
    reset = reset or TerrainResetB200(env["ml"], env["floor"], env["terrain"], env["cx"], env["cy"])
    sim = _sim(n, seed, (env["hf"].shape[0] * 0.1, env["hf"].shape[1] * 0.1))
    task.reset_task(torch.arange(n, device=DEV), sim["root_states"])          # the initial waypoints, from the roots
    task.traj_verts[::11, :, 0:2] = sim["root_states"][::11, None, 0:2]      # envs at the episode's end stay on their waypoints
    g = torch.Generator().manual_seed(seed + 1)
    freeze = torch.zeros(69, dtype=torch.uint8)
    freeze[[9, 10, 11, 66, 67, 68]] = 1
    drv = TerrainStepsB200(task, reset, _policy(), PulseVAE(device=DEV, with_critic=False, seed=1), sim, horizon=T,
                           pd_offset=torch.randn(69, generator=g).to(DEV), pd_scale=(0.5 + torch.rand(69, generator=g)).to(DEV),
                           pd_freeze=freeze.to(DEV), use_graphs=use_graphs, reset_seed=3)
    drv.first_observation()
    return drv


def _state(drv):
    s = drv.sim
    out = {k: getattr(drv, k) for k in ("obses", "obs_carry", "actions", "mus", "neglogp", "values", "next_values", "rewards", "dones", "pd_tar",
                                        "reset_buf", "terminate_buf")}
    out.update({k: s[k] for k in ("body_state", "root_all", "dof_state", "contact_forces", "progress_buf", "sampled_motion_ids", "motion_start_times")})
    out["traj_verts"] = drv.task.traj_verts
    return out


def _assert_same(a, b, what=""):
    sa, sb = _state(a), _state(b)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f"{what}: {k} differs"


def _obs(n, seed=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, 1402, generator=g) * 1.5).to(DEV)


# ------------------------------------------------------------------------------------------------ 1. SeptPolicy rollout side
def test_sept_heads_and_critic_values_into():
    n = 1027
    pol = _policy()
    obs = _obs(n)
    mus = torch.zeros(n, 3, 32, device=DEV)
    value = pol.heads_into(obs, mus=mus[:, 1], side=torch.cuda.Stream(DEV)).clone()
    ref = pol.act(obs, eps=torch.zeros(n, 32, device=DEV))
    ref_value = pol.critic._workspace(n, False)["out"].clone()                 # act()'s normalised value
    assert torch.equal(mus[:, 1], ref["mus"]) and float(mus[:, [0, 2]].abs().max()) == 0
    assert torch.equal(value, ref_value)
    assert torch.equal(pol.value_rms.unnormalize(value), ref["values"])
    terminate = (torch.arange(n, device=DEV) % 5 == 0).long()
    outs = []
    for slot in (0, 1):
        out = torch.full((n, 1), 9.0, device=DEV)
        pol.critic_values_into(obs, out.view(-1), terminate=terminate, slot=slot)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    expect = torch.zeros(n, 1, device=DEV)
    pol._value_post(ref_value, terminate, expect.view(-1))
    assert torch.equal(outs[1], expect)
    torch.testing.assert_close(outs[1], ref["values"] * (1 - terminate.float()).view(-1, 1), atol=1e-6, rtol=1e-6)
    assert float(outs[1][terminate.bool()].abs().max()) == 0 and float(outs[1].abs().max()) > 0


def test_sept_act_into_matches_act():
    n = 1027
    pol = _policy()
    obs = _obs(n, seed=4)
    eps = torch.randn(n, 32, generator=torch.Generator().manual_seed(6)).to(DEV)
    actions, nlp, mus, values = torch.zeros(n, 2, 32, device=DEV), torch.zeros(n, 2, device=DEV), torch.zeros(n, 2, 32, device=DEV), torch.zeros(2, n, 1, device=DEV)
    off, sc, pd = torch.randn(32, device=DEV), torch.rand(32, device=DEV) + 0.5, torch.zeros(n, 32, device=DEV)
    pol.act_into(obs, actions=actions[:, 1], neglogp=nlp[:, 1], mus=mus[:, 1], values=values[1], pd=(off, sc, pd), eps=eps, side=torch.cuda.Stream(DEV))
    ref = pol.act(obs, eps=eps)
    torch.testing.assert_close(mus[:, 1], ref["mus"], atol=0, rtol=0)
    torch.testing.assert_close(actions[:, 1], ref["actions"], atol=1e-6, rtol=1e-6)
    torch.testing.assert_close(nlp[:, 1], ref["neglogpacs"], atol=2e-4, rtol=1e-5)
    torch.testing.assert_close(values[1], ref["values"], atol=1e-6, rtol=1e-6)
    torch.testing.assert_close(pd, off + sc * actions[:, 1], atol=1e-6, rtol=1e-6)


# ------------------------------------------------------------------------------------------------ 2. pulse_terrain_rollout_step
@pytest.mark.parametrize("power", [False, True])
def test_rollout_step_equals_advance_then_step(env, power):
    n, t = 1027, 1
    drv = _driver(env, n, power=power)
    task, s = drv.task, drv.sim
    progress0 = s["progress_buf"].clone()
    s["progress_buf"].add_(1)                                                 # the plain path: advance, then the task's own step
    task.post_physics_step(s["body_state"], s["root_states"], s["progress_buf"], s["contact_forces"], s["dof_force"], s["dof_vel"])
    s["progress_buf"].copy_(progress0)
    drv._env_step(t)
    assert torch.equal(s["progress_buf"], progress0 + 1)
    assert torch.equal(drv.obses[:, t + 1], task.obs_buf) and float(drv.obses[:, t].abs().max()) == 0
    assert torch.equal(drv.rewards[t], task.rew_buf)
    assert torch.equal(drv.reset_buf, task.reset_buf) and torch.equal(drv.terminate_buf, task._terminate_buf)
    assert torch.equal(drv.dones[t], task.reset_buf.float())
    ended = (progress0 + 1 >= task.max_episode_length - 1) & (drv.terminate_buf == 0) & (drv.reset_buf == 1)
    assert int(ended.sum()) > 0 and 0 < int(drv.terminate_buf.sum()) < n and bool((drv.terminate_buf[::7] == 1).all())
    if power:
        assert not torch.equal(task.rew_buf, task.reward_raw[:, 0])


# ------------------------------------------------------------------------------------------------ 2b. separate heightfield uploads
def test_driver_from_separate_uploads_of_one_map(env):
    """The wiring of INTEGRATION.md: the task's TerrainB200 and the reset's come from two `from_reference` calls on one reference
    `Terrain`, i.e. two device copies of the map.  The driver accepts them and computes what it computes over one shared copy; a
    map that differs in one cell is refused."""
    from types import SimpleNamespace as NS

    from pulse_b200 import PulseError
    from pulse_b200.terrain import TerrainB200
    from pulse_b200.terrain_reset import TerrainResetB200
    from pulse_b200.terrain_rollout import TerrainStepsB200
    n = 1027
    ref = NS(heightsamples=env["hf"].numpy(), horizontal_scale=0.1, vertical_scale=0.005, coord_x_scale=env["cx"].numpy(),
             coord_y_scale=env["cy"].numpy())
    task_terrain = TerrainB200.from_reference(ref, DEV, "trimesh")
    reset = TerrainResetB200.from_reference(ref, env["ml"], env["floor"], "trimesh")
    assert task_terrain.heightfield.data_ptr() != reset.terrain.heightfield.data_ptr()
    a = _driver(env, n, T=3, use_graphs=False, task_terrain=task_terrain, reset=reset)
    b = _driver(env, n, T=3, use_graphs=False)
    resets = 0.0
    for _ in range(2):
        a.play_steps()
        b.play_steps()
        _assert_same(a, b, "separate uploads")
        resets += float(a.dones.sum())
    assert resets > 0
    bumped = env["hf"].clone()
    bumped[150, 250] += 1
    with pytest.raises(PulseError, match="different heightfields"):
        TerrainStepsB200(a.task, TerrainResetB200(env["ml"], env["floor"], TerrainB200(bumped, device=DEV), env["cx"], env["cy"]), a.policy,
                         a.vae, a.sim)


# ------------------------------------------------------------------------------------------------ 2c. the Philox keying of a step
def test_philox_blocks_are_the_kernels_draws(env):
    """`philox_blocks` names the blocks the kernels read.  Regenerated on the host (tests/philox_ref.py) and injected, the reset's
    clip, start-time and location draws and the waypoint draws reproduce the driver's Philox step bit for bit; the latent noise the
    driver drew equals the host's Box-Muller of the named blocks (within the tolerance of the kernel's __logf / __sincosf)."""
    import ctypes as C

    import numpy as np

    from pulse_b200 import _lib
    from pulse_b200.terrain_rollout import philox_blocks
    from tests.philox_ref import box_muller, philox4x32_10, u01
    n, t, off = 1027, 3, 64
    a = _driver(env, n, use_graphs=False)
    b = _driver(env, n, use_graphs=False)
    for d in (a, b):
        d.policy.rng_offset.fill_(off)
        d.reset_buf[::3] = 1
    a._reset(t)
    a._reset_obs(t)

    blocks = [philox_blocks(e, t, off) for e in range(n)]
    S = _lib.TRAJ_VERTS - 1

    def words(key, rows):
        seed = b.reset_seed if key == "reset" else b.policy.rng_seed
        assert all(k == key for k, _, _ in rows)
        return philox4x32_10(seed, [i for _, i, _ in rows], [c for _, _, c in rows])

    x, y, z, _ = words("reset", [bl[0] for bl in blocks])
    L = b.reset.num_locations
    dev = lambda v, dt: torch.from_numpy(np.ascontiguousarray(v)).to(DEV, dt)
    phase, motion_u = dev(u01(x), torch.float32), dev(u01(y), torch.float32)
    loc = dev(((z * np.uint64(L)) >> np.uint64(32)).astype(np.int64), torch.int64)
    tw = np.stack(words("reset", [r for bl in blocks for r in bl[1:_lib.TRAJ_VERTS + 1]])).reshape(4, n, _lib.TRAJ_VERTS)
    rand = np.zeros((n, _lib.TRAJ_DRAWS), dtype=np.float32)
    for j in range(4):                                           # block k < S: turn, sharp turn, coin, speed change of segment k
        rand[:, j * S:(j + 1) * S] = u01(tw[j][:, :S])
    rand[:, 4 * S], rand[:, 4 * S + 1] = u01(tw[0][:, S]), u01(tw[1][:, S])     # block S: initial heading and speed

    s = b.sim
    b.reset_ws = ws = b.reset.reset_envs(root_states=s["root_states"], dof_pos=s["dof_pos"], dof_vel=s["dof_vel"], rigid_body_state=s["body_state"],
                                         progress_buf=s["progress_buf"], sampled_motion_ids=s["sampled_motion_ids"],
                                         motion_start_times=s["motion_start_times"], reset_buf=b.reset_buf, contact_forces=s["contact_forces"],
                                         actor_ids=s["actor_ids"], motion_u=motion_u, phase=phase, loc_ids=loc)
    args = b._step_args(_lib.STEP_OBS, b.obses[:, t], b.rewards[t])
    args.env_ids, args.env_count = ws["env_list"].data_ptr(), ws["count"].data_ptr()
    b._launch("pulse_terrain_step", C.byref(args), n)
    b.reset.reset_task(b.task, s["root_states"], rand=dev(rand, torch.float32))
    _assert_same(a, b, "injected draws")
    assert torch.equal(a.reset_ws["loc_ids"], ws["loc_ids"]) and int(ws["count"]) == len(range(0, n, 3))

    a._act(t)
    pw = words("policy", [r for bl in blocks for r in bl[_lib.TRAJ_VERTS + 1:]])
    n0, n1 = (w.reshape(n, -1) for w in box_muller(pw[0], pw[1]))
    eps = np.empty((n, 32))
    eps[:, 0::2], eps[:, 1::2] = n0, n1
    drawn = (a.actions[:, t] - a.mus[:, t]) / torch.exp(a.policy.logstd)
    err = (drawn.double().cpu() - torch.from_numpy(eps)).abs()
    assert float(err.max()) < 2e-3 and float(err.mean()) < 2e-5, (float(err.max()), float(err.mean()))


# ------------------------------------------------------------------------------------------------ 3. composition from public calls
def test_eager_steps_equal_the_public_calls(env):
    """Three eager driver steps against the same steps composed from TerrainResetB200.reset_envs / observe / reset_task,
    SeptPolicy.act, PulseVAE.compute_z_actions, pulse_pd_targets and the advanced step, taking the driver's sampled actions as given."""
    from pulse_b200.terrain import PedestrianTerrainTaskB200
    from pulse_b200.vae import pd_targets
    n, T = 1027, 3
    drv = _driver(env, n, T=T, use_graphs=False)
    pol, vae, reset = drv.policy, drv.vae, drv.reset
    s2 = {k: v.clone() for k, v in drv.sim.items() if k in ("body_state", "root_all", "dof_state", "contact_forces", "progress_buf",
                                                           "sampled_motion_ids", "motion_start_times", "dof_force", "actor_ids")}
    s2.update(root_states=s2["root_all"][:, 0], dof_pos=s2["dof_state"][:, :69, 0], dof_vel=s2["dof_state"][:, :69, 1])
    task2 = PedestrianTerrainTaskB200(n, device=DEV, terrain=env["terrain"], seed=11)
    task2.traj_verts.copy_(drv.task.traj_verts)
    off0 = pol.rng_offset.clone()
    snap = []
    drv.physics = lambda t: snap.append((drv.z_actions.clone(), drv.pd_tar.clone()))
    drv.play_steps()

    task2.compute_observations(s2["body_state"], s2["root_states"], s2["progress_buf"])
    obs = task2.obs_buf.clone()
    assert torch.equal(obs, drv.obses[:, 0])
    resets = 0
    for t in range(T):
        ws = reset.reset_envs(root_states=s2["root_states"], dof_pos=s2["dof_pos"], dof_vel=s2["dof_vel"], rigid_body_state=s2["body_state"],
                              progress_buf=s2["progress_buf"], sampled_motion_ids=s2["sampled_motion_ids"],
                              motion_start_times=s2["motion_start_times"], reset_buf=task2.reset_buf, contact_forces=s2["contact_forces"],
                              actor_ids=s2["actor_ids"], seed=drv.reset_seed, offset=t, offset_dev=off0)
        ids = ws["env_list"][:int(ws["count"].item())].clone()
        resets += ids.numel()
        reset.observe(task2, s2["body_state"], s2["root_states"], s2["progress_buf"])
        obs[ids] = task2.obs_buf[ids]
        reset.reset_task(task2, s2["root_states"], seed=drv.reset_seed, offset=t, offset_dev=off0)
        assert torch.equal(obs, drv.obses[:, t]), f"step {t}: observation"
        ref = pol.act(obs, eps=torch.zeros(n, 32, device=DEV))
        assert torch.equal(ref["mus"], drv.mus[:, t]), f"step {t}: mus"
        torch.testing.assert_close(drv.values[t], ref["values"], atol=1e-6, rtol=1e-6)
        dec = vae.compute_z_actions(obs, drv.actions[:, t])
        assert torch.equal(dec, snap[t][0]), f"step {t}: decoder output"
        assert torch.equal(pd_targets(dec, drv.pd[0], drv.pd[1], freeze=drv.pd_freeze), snap[t][1]), f"step {t}: PD targets"
        s2["progress_buf"].add_(1)
        task2.post_physics_step(s2["body_state"], s2["root_states"], s2["progress_buf"], s2["contact_forces"], s2["dof_force"], s2["dof_vel"])
        obs = task2.obs_buf.clone()
        # the reset envs' rows of obses[:, t+1] are rewritten by the reset of step t+1 (checked above, at the next step)
        kept = task2.reset_buf == 0 if t + 1 < T else torch.ones(n, dtype=torch.bool, device=DEV)
        assert torch.equal(obs[kept], drv._next_obs(t)[kept]), f"step {t}: next observation"
        assert torch.equal(task2.rew_buf, drv.rewards[t]) and torch.equal(task2.reset_buf.float(), drv.dones[t])
        nv = pol.critic_values(obs) * (1 - task2._terminate_buf.float()).view(-1, 1)
        torch.testing.assert_close(drv.next_values[t], nv, atol=1e-6, rtol=1e-6)
    assert torch.equal(task2.reset_buf, drv.reset_buf) and torch.equal(task2._terminate_buf, drv.terminate_buf)
    for k in ("body_state", "root_all", "dof_state", "contact_forces", "progress_buf", "sampled_motion_ids", "motion_start_times"):
        assert torch.equal(s2[k], drv.sim[k]), k
    assert torch.equal(task2.traj_verts, drv.task.traj_verts)
    assert resets > 0


# ------------------------------------------------------------------------------------------------ 4. horizon: graphs + streams vs eager
@pytest.mark.parametrize("n", [1027, 8192])
def test_horizon_graph_equals_sequential(env, n):
    T = 4
    a = _driver(env, n, T=T, use_graphs=True)
    b = _driver(env, n, T=T, use_graphs=False)
    _assert_same(a, b, "initial")
    progress0 = b.sim["progress_buf"].clone()
    for use in ("eager", "capture", "replay"):
        a.play_steps()
        b.play_steps()
        _assert_same(a, b, use)
        if use == "eager":                  # step 0 resets the envs with a contact force (early termination) and those at the episode's end
            contact = b.dones[0][::7] == 1
            ended = (b.dones[0] == 1) & (progress0 + 1 >= b.task.max_episode_length - 1)
            assert bool(contact.all()) and int(ended.sum()) >= n // 11 and float(b.dones.sum()) < T * n / 2
        a.finish()
        b.finish()
        assert torch.equal(a.adv, b.adv) and torch.equal(a.ret, b.ret)
    assert isinstance(a._graphs[("horizon",)], torch.cuda.CUDAGraph)
    assert bool(torch.isfinite(a.obses).all()) and bool(torch.isfinite(a.next_values).all())


# ------------------------------------------------------------------------------------------------ 5. hook mode
def test_hooks_run_as_graph_segments(env):
    n, T = 1027, 3
    a = _driver(env, n, T=T, use_graphs=True)
    b = _driver(env, n, T=T, use_graphs=False)

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
    b.refresh = lambda t, ws: None
    for use in ("eager", "capture", "replay"):
        a.play_steps()
        b.play_steps()
        _assert_same(a, b, use)
    assert sum(int(c) for c in counts) > 0
    assert all(isinstance(a._graphs[(seg, t)], torch.cuda.CUDAGraph) for seg in ("reset", "act", "post") for t in range(T))


# ------------------------------------------------------------------------------------------------ 6-7. finish, train_epoch, no syncs
def test_finish_and_train_epoch(env):
    from pulse_b200.rollout import discount_values
    n, T = 1024, 4
    a = _driver(env, n, T=T, use_graphs=True)
    b = _driver(env, n, T=T, use_graphs=False)
    for _ in range(3):
        for d in (a, b):
            d.play_steps()
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
        for name in ("running_mean", "running_var"):
            torch.testing.assert_close(getattr(a.policy.obs_rms, name), getattr(pol.obs_rms, name), rtol=1e-12, atol=1e-15)
            getattr(pol.obs_rms, name).copy_(getattr(a.policy.obs_rms, name))
        pol.obs_rms._refresh()
    assert float(stats.abs().sum()) > 0
    with pytest.raises(Exception):
        a.train_epoch(minibatch=1000)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a.play_steps()
        a.finish()
        a.train_epoch(mini_epochs=2, minibatch=1024)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
