"""The drop-in layer EXECUTED: `HumanoidImB200Mixin` and `AMPAgentB200Mixin` mixed in front of stand-in base classes that carry the
reference's attribute / method contract (tests/standins.py; checked against names recorded from the reference sources by
tests/test_boundary_cpu.py).

  task  : Humanoid.post_physics_step -> _compute_reward -> _compute_reset -> _compute_observations -> AMP history + observation
          (humanoid.py:1315-1346, humanoid_amp.py:194-210) against the oracle; the getup recovery masking (humanoid_im_getup.py:203-210)
  agent : get_action_values / _eval_critic / _calc_amp_rewards / discount_values / prepare_dataset / calc_gradients through the mixin,
          then a checkpoint ROUND TRIP through `self.model.state_dict()` / `optimizer.state_dict()` / the normaliser modules
          (common_agent.py:142-150 saves exactly those)."""
import copy

import pytest
import torch

from tests.helpers import exact_step_inputs, exact_tables
from tests.standins import StandInAMPAgent, StandInHumanoidIm

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mlib(tb):
    from pulse_b200.motion_lib import MotionLibB200
    return MotionLibB200.from_tables({k: getattr(tb, k) for k in ("gts", "grs", "lrs", "gvs", "gavs", "dvs", "motion_aa", "lengths", "num_frames", "dt",
                                                                   "length_starts")}, device=DEV)


@pytest.mark.parametrize("getup", [False, True])
def test_task_mixin_post_physics_step_matches_oracle(getup):
    from oracle import pulse_oracle as po
    from pulse_b200.humanoid_im import HumanoidImB200Mixin

    class HumanoidImB200(HumanoidImB200Mixin, StandInHumanoidIm):
        pass

    n = 389
    tb = exact_tables(41, seed=8)
    z, _ = exact_step_inputs(tb, n, seed=9)
    task = HumanoidImB200(_mlib(tb), z, DEV, getup=getup)
    rec = None
    if getup:
        g = torch.Generator().manual_seed(1)
        rec = (torch.rand(n, generator=g) < 0.25).int() * 40
        task._recovery_counter.copy_(rec.to(DEV))
    amp0 = torch.randn(n, 10, 196, device=DEV)
    task._amp_obs_buf.copy_(amp0)
    task.post_physics_step()
    torch.cuda.synchronize()
    ref = po.humanoid_im_step(tb, po.ImStepConfig(), z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"], z["start_times"],
                              z["start_offset"], z["global_offset"], z["cycle_counter"], z["reset_buf_in"], recovery_counter=rec)
    assert torch.equal(task.reset_buf.cpu(), ref["reset_buf"]) and torch.equal(task._terminate_buf.cpu(), ref["terminate_buf"])
    assert torch.equal(task.progress_buf.cpu(), ref["progress_buf"] if getup else z["progress_buf"])
    torch.testing.assert_close(task.obs_buf.cpu(), ref["obs_buf"], atol=1e-4, rtol=0)
    torch.testing.assert_close(task.self_obs_buf.cpu(), ref["obs_buf"][:, :358], atol=1e-4, rtol=0)
    torch.testing.assert_close(task.rew_buf.cpu(), ref["rew_buf"], atol=1e-4, rtol=0)
    torch.testing.assert_close(task.reward_raw.cpu(), ref["reward_raw"], atol=1e-4, rtol=0)
    torch.testing.assert_close(task.ref_body_pos.cpu(), ref["ref_body_pos"], atol=1e-5, rtol=0)
    amp_ref = po.amp_obs_step(amp0.cpu(), z["body_state"], z["dof_pos"], z["dof_vel"])
    torch.testing.assert_close(task._amp_obs_buf.cpu(), amp_ref, atol=1e-4, rtol=0)
    assert task.extras["amp_obs"].shape == (n, 1960)
    # reset-time observation of a subset through the same override (humanoid.py:574-587 -> _compute_observations(env_ids))
    ids = torch.tensor([3, 77, 388], device=DEV)
    before = task.obs_buf.clone()
    task.obs_buf[ids] = -7.0
    task._compute_observations(ids)
    torch.cuda.synchronize()
    if not getup:       # recovering envs take their observation one step earlier in the fused call; the subset call re-queries at progress + 1
        torch.testing.assert_close(task.obs_buf, before, atol=1e-6, rtol=0)


@pytest.mark.parametrize("obs_v,track,fut", [(7, [13, 18, 23], True), (9, [0, 4, 8, 13, 18, 23], False), (1, [0, 4, 8, 13, 18, 23], True), (3, list(range(24)), False)])
def test_task_mixin_general_observation_configurations(obs_v, track, fut):
    """SURVEY 8f-4 through the drop-in layer: a task configured with another observation version / a tracked-body subset / a fut_tracks
    window (env_pulse_im.yaml-style 3-point tracking, humanoid_im.py:708-851) -- reward and reset still come from the fused kernel, the
    observation is [self obs | general task-observation kernel]."""
    from oracle import pulse_oracle as po
    from pulse_b200.humanoid_im import HumanoidImB200Mixin

    class HumanoidImB200(HumanoidImB200Mixin, StandInHumanoidIm):
        pass

    n = 389
    tb = exact_tables(41, seed=8)
    z, _ = exact_step_inputs(tb, n, seed=9)
    task = HumanoidImB200(_mlib(tb), z, DEV)
    task.obs_v, task._track_bodies_id, task._fut_tracks = obs_v, torch.tensor(track, device=DEV), fut
    task._num_traj_samples, task._traj_sample_timestep, task._has_upright_start = 3, 0.5, True
    task.post_physics_step = lambda: (task.progress_buf.add_(1), task._compute_reward(None), task._compute_reset(), task._compute_observations())
    task.post_physics_step()
    torch.cuda.synchronize()
    ref = po.humanoid_im_step(tb, po.ImStepConfig(), z["body_state"], z["dof_vel"], z["dof_force"], z["progress_buf"], z["motion_ids"], z["start_times"],
                              z["start_offset"], z["global_offset"], z["cycle_counter"], z["reset_buf_in"])
    assert torch.equal(task.reset_buf.cpu(), ref["reset_buf"]) and torch.equal(task._terminate_buf.cpu(), ref["terminate_buf"])
    torch.testing.assert_close(task.rew_buf.cpu(), ref["rew_buf"], atol=1e-4, rtol=0)
    torch.testing.assert_close(task.obs_buf[:, :358].cpu(), ref["obs_buf"][:, :358], atol=1e-4, rtol=0)
    T = 3 if fut else 1
    dt = po.STEP_DT
    t0 = (z["progress_buf"] + 1) * dt
    times = (t0[:, None] + (torch.arange(T) * 0.5)[None, :] + z["start_times"][:, None] + z["start_offset"][:, None]).reshape(-1) if T > 1 \
        else t0 + z["start_times"] + z["start_offset"]
    q = po.motion_state(tb, z["motion_ids"].repeat_interleave(T), times.float(), z["global_offset"].repeat_interleave(T, dim=0))
    bs, tr = z["body_state"], torch.tensor(track)
    want = po.imitation_obs(obs_v, bs[:, 0, 0:3], bs[:, 0, 3:7], bs[:, tr, 0:3], bs[:, tr, 3:7], bs[:, tr, 7:10], bs[:, tr, 10:13],
                            q["rg_pos"][:, tr], q["rb_rot"][:, tr], q["body_vel"][:, tr], q["body_ang_vel"][:, tr], T, True)
    torch.testing.assert_close(task.obs_buf[:, 358:358 + want.shape[1]].cpu(), want, atol=1e-4, rtol=0)
    torch.testing.assert_close(task.ref_body_pos.cpu(), q["rg_pos"].view(n, T, 24, 3)[:, 0], atol=1e-5, rtol=0)
    # reset-time observation of a subset through the same override
    ids = torch.tensor([3, 77, 388], device=DEV)
    before = task.obs_buf.clone()
    task.obs_buf[ids] = -7.0
    task._compute_observations(ids)
    torch.cuda.synchronize()
    torch.testing.assert_close(task.obs_buf[:, :358 + want.shape[1]], before[:, :358 + want.shape[1]], atol=1e-6, rtol=0)


def test_task_mixin_reset_envs_matches_oracle():
    """`_reset_envs(env_ids)` through the mixin (one fused launch + the reference's own gym setters / refresh / observation call) against
    the oracle's restatement of the reference's reset chain, with the start-time draws taken from torch's generator exactly as
    `sample_time_interval` takes them."""
    from oracle import pulse_oracle as po
    from pulse_b200.humanoid_im import HumanoidImB200Mixin

    class HumanoidImB200(HumanoidImB200Mixin, StandInHumanoidIm):
        pass

    n = 389
    tb = exact_tables(41, seed=8)
    z, _ = exact_step_inputs(tb, n, seed=9)
    task = HumanoidImB200(_mlib(tb), z, DEV)
    g = torch.Generator().manual_seed(2)
    task._amp_obs_buf.copy_(torch.randn(n, 10, 196, generator=g).to(DEV))
    task.obs_buf.copy_(torch.randn(n, 934, generator=g).to(DEV))
    task._humanoid_root_states.copy_(torch.randn(n, 13, generator=g).to(DEV))
    task._terminate_buf.copy_((torch.rand(n, generator=g) < 0.3).long().to(DEV))
    env_ids = torch.nonzero(torch.rand(n, generator=g) < 0.2).flatten().to(DEV)
    st = {"motion_ids": task._sampled_motion_ids, "start_times": task._motion_start_times, "start_offset": task._motion_start_times_offset,
          "global_offset": task._global_offset, "cycle_counter": task._cycle_counter, "progress_buf": task.progress_buf,
          "reset_buf": task.reset_buf, "terminate_buf": task._terminate_buf, "root_states": task._humanoid_root_states,
          "dof_pos": task._dof_pos, "dof_vel": task._dof_vel, "body_state": task._rigid_body_state_reshaped[:, :24],
          "contact_forces": task._contact_forces[:, :24], "amp_obs_buf": task._amp_obs_buf, "obs_buf": task.obs_buf,
          "dof_force": task.dof_force_tensor}
    st = {k: v.detach().cpu().clone().contiguous() for k, v in st.items()}
    torch.manual_seed(77)
    draws = torch.rand(env_ids.shape, device=DEV)                     # what sample_time_interval would draw for these envs
    phase = torch.zeros(n)
    phase[env_ids.cpu()] = draws.cpu()
    torch.manual_seed(77)
    task._reset_envs(env_ids)
    torch.cuda.synchronize()
    exp = po.reset_envs(tb, po.ImStepConfig(), st, env_ids.cpu(), phase)
    ids = env_ids.cpu()
    assert torch.equal(task.progress_buf.cpu(), exp["progress_buf"]) and torch.equal(task.reset_buf.cpu(), exp["reset_buf"])
    assert torch.equal(task._terminate_buf.cpu(), exp["terminate_buf"]) and torch.equal(task._cycle_counter.cpu(), exp["cycle_counter"])
    torch.testing.assert_close(task._motion_start_times.cpu(), exp["start_times"], atol=0, rtol=0)
    torch.testing.assert_close(task._motion_start_times_offset.cpu(), exp["start_offset"], atol=0, rtol=0)
    torch.testing.assert_close(task._global_offset.cpu(), exp["global_offset"], atol=0, rtol=0)
    torch.testing.assert_close(task._humanoid_root_states.cpu(), exp["root_states"], atol=1e-5, rtol=0)
    torch.testing.assert_close(task._dof_pos.cpu(), exp["dof_pos"], atol=1e-4, rtol=1e-4)
    torch.testing.assert_close(task._dof_vel.cpu(), exp["dof_vel"], atol=1e-4, rtol=0)
    # the rigid bodies of the reset envs survive gym's refresh through the reference's _reset_rb_* restore; the others are the simulator's
    torch.testing.assert_close(task._rigid_body_state_reshaped[:, :24].cpu(), exp["body_state"], atol=1e-5, rtol=0)
    assert float(task._contact_forces[env_ids].abs().max()) == 0.0 and float(task._contact_forces.sum()) == 3 * 26 * (n - len(ids))
    torch.testing.assert_close(task._amp_obs_buf.cpu(), exp["amp_obs_buf"], atol=1e-4, rtol=0)
    torch.testing.assert_close(task.obs_buf.cpu(), exp["obs_buf"], atol=1e-4, rtol=0)
    assert [c[0] for c in task.gym_calls] == ["set_actor_root_state_tensor_indexed", "set_dof_state_tensor_indexed"]
    assert torch.equal(task.gym_calls[0][1].cpu(), (2 * ids).to(torch.int32)) and task.gym_calls[0][2] == len(ids)
    assert torch.equal(task._reset_ref_motion_times.cpu(), exp["start_times"][ids]) and task._state_reset_happened is False
    # an empty list and the non-reference initialisations go back to the reference implementation
    with pytest.raises(AssertionError, match="reference reset path"):
        task._reset_envs(env_ids[:0])


def _agent(seed=0, **kw):
    from pulse_b200.agent_mixins import AMPAgentB200Mixin

    class IMAmpAgentB200(AMPAgentB200Mixin, StandInAMPAgent):
        pass

    return IMAmpAgentB200(task=None, device=DEV, seed=seed, **kw)


def _minibatch(agent, M=2048, seed=5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    obs = torch.randn(M, 934, device=DEV, generator=g)
    res = agent.get_action_values({"obs": obs})
    n = agent._amp_minibatch_size
    amp = [torch.randn(n, 1960, device=DEV, generator=g) for _ in range(3)]
    return {"obs": obs, "actions": res["actions"].clone(), "old_logp_actions": res["neglogpacs"].clone(), "mu": res["mus"].clone(),
            "advantages": torch.randn(M, device=DEV, generator=g), "returns": torch.randn(M, device=DEV, generator=g),
            "amp_obs": amp[0], "amp_obs_replay": amp[1], "amp_obs_demo": amp[2]}, res


def test_agent_mixin_methods_and_checkpoint_round_trip():
    agent = _agent(seed=1)
    agent._amp_minibatch_size = 512
    init = copy.deepcopy(agent.model.state_dict())
    batch, res = _minibatch(agent)
    M = batch["obs"].shape[0]
    assert res["actions"].shape == (M, 69) and res["values"].shape == (M, 1) and res["neglogpacs"].shape == (M,) and res["rnn_states"] is None
    v = agent._eval_critic({"obs": batch["obs"]})
    torch.testing.assert_close(v, res["values"], atol=1e-5, rtol=1e-5)           # same critic, same (identity) value statistics
    r = agent._calc_amp_rewards(batch["amp_obs"].view(16, 32, 1960))
    assert r["disc_rewards"].shape == (16, 32, 1) and bool((r["disc_rewards"] >= 0).all())
    T, N = 8, 64
    adv = agent.discount_values(torch.zeros(T, N, device=DEV), torch.randn(T, N, 1, device=DEV), torch.randn(T, N, 1, device=DEV), torch.randn(T, N, 1, device=DEV))
    assert adv.shape == (T, N, 1)
    # prepare_dataset keeps value_mean_std the owner and mirrors it into the device library
    agent.prepare_dataset({"values": torch.randn(4096, 1, device=DEV) * 3 + 1, "returns": torch.randn(4096, 1, device=DEV) * 3 + 1})
    pol = agent._pulse_policy()
    torch.testing.assert_close(pol.value_rms.running_mean, agent.value_mean_std.running_mean.reshape(-1))
    torch.testing.assert_close(pol.value_rms.running_var, agent.value_mean_std.running_var.reshape(-1))
    assert float(pol.value_rms.count) == float(agent.value_mean_std.count) == 1 + 2 * 4096
    # two training steps through calc_gradients
    for _ in range(2):
        agent.calc_gradients(batch)
    tr = agent.train_result
    for k in ("actor_loss", "critic_loss", "b_loss", "kl", "actor_clip_frac", "disc_loss", "disc_agent_acc", "disc_demo_acc", "disc_agent_logit",
              "disc_demo_logit", "disc_grad_penalty", "disc_logit_loss"):
        assert k in tr and torch.isfinite(torch.as_tensor(tr[k]).float()).all(), k
    # ---- save: what rl_games serialises must be the TRAINED state ---------------------------------------------------------------
    w = copy.deepcopy(agent.get_full_state_weights())
    sd = w["model"]
    assert not torch.equal(sd["a2c_network.actor_mlp.0.weight"], init["a2c_network.actor_mlp.0.weight"])       # trained, not the initial weights
    assert not torch.equal(sd["a2c_network._disc_mlp.2.bias"], init["a2c_network._disc_mlp.2.bias"])
    torch.testing.assert_close(sd["a2c_network.mu.weight"], pol.actor.layers[-1].weight[:, :512], atol=0, rtol=0)
    assert float(w["running_mean_std"]["count"]) == 1 + 2 * M and float(w["amp_input_mean_std"]["count"]) == 1 + 2 * 3 * 512
    st = w["optimizer"]["state"]
    assert len(st) > 0 and all(float(s["step"]) == 2 for s in st.values()) and any(float(s["exp_avg"].abs().max()) > 0 for s in st.values())
    # ---- restore into a fresh agent and continue: identical to continuing in the original ------------------------------------------
    other = _agent(seed=99)
    other._amp_minibatch_size = 512
    other.get_action_values({"obs": batch["obs"]})            # builds its device copy from DIFFERENT weights first
    other.set_full_state_weights(w)
    pol2 = other._pulse_policy()
    assert pol2 is not pol
    torch.testing.assert_close(pol2.flat.params, pol.flat.params, atol=0, rtol=0)
    torch.testing.assert_close(pol2.flat.exp_avg, pol.flat.exp_avg, atol=0, rtol=0)
    torch.testing.assert_close(pol2.flat.exp_avg_sq, pol.flat.exp_avg_sq, atol=0, rtol=0)
    assert int(pol2.flat.step) == 2
    torch.testing.assert_close(pol2.obs_rms.running_var, pol.obs_rms.running_var, atol=0, rtol=0)
    torch.testing.assert_close(pol2.disc.rms.running_mean, pol.disc.rms.running_mean, atol=0, rtol=0)
    torch.testing.assert_close(pol2.value_rms.running_mean, pol.value_rms.running_mean, atol=0, rtol=0)
    agent.calc_gradients(batch)
    other.calc_gradients(batch)
    torch.cuda.synchronize()
    # same arithmetic from the same state; the weight-gradient reductions add in a different order run to run (fp32, ~1e-7 relative)
    torch.testing.assert_close(pol2.flat.params, pol.flat.params, atol=1e-6, rtol=1e-5)
    assert float((pol2.flat.params - pol.flat.params).abs().max()) < 1e-4


def test_agent_mixin_reads_network_shape_from_the_model():
    """pulse_z_task.yaml-style policy (2048-1024-512 SiLU): units / activation come from the model, not from defaults."""
    import tests.standins as si
    agent = _agent(seed=3, obs=361, actions=32, units=(2048, 1024, 512), amp=1960, disc_units=(1024, 512))
    agent.model.a2c_network.actor_mlp = si.mlp((361, 2048, 1024, 512), torch.nn.SiLU).to(DEV)
    agent.model.a2c_network.critic_mlp = si.mlp((361, 2048, 1024, 512), torch.nn.SiLU).to(DEV)
    pol = agent._pulse_policy()
    assert [l.N for l in pol.actor.layers] == [2048, 1024, 512, 32] and pol.actor.act == "silu" and pol.obs_size == 361
    res = agent.get_action_values({"obs": torch.randn(256, 361, device=DEV)})
    x = torch.clamp(torch.randn(1), -5, 5)  # noqa: F841
    ref_mu = agent.model.a2c_network.mu(agent.model.a2c_network.actor_mlp(torch.clamp(_last_obs(agent, res), -5, 5)))
    torch.testing.assert_close(res["mus"], ref_mu, atol=3e-2, rtol=3e-2)


def _last_obs(agent, res):
    """the observation batch of the last get_action_values call, normalised with the (identity) statistics"""
    pol = agent._pulse_policy()
    return pol._buf(res["mus"].shape[0], False)["x"][:, :pol.obs_size].float()
