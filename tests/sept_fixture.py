"""Weights and minibatches of the amp_sept (pedestrian terrain) policy fixture, regenerated from integer draws on a seeded CPU generator
(exact on every host) by the golden generator (tests/golden/make_golden_sept.py) and by the tests.  The production-width net has 9 M
parameters, so only a float64 checksum of what was generated is stored next to the reference's outputs."""
import torch

from tests.helpers import _approx_normal, _uniform_pm1

# (a) shrunk widths: every parameter gradient is stored; (b) pulse_z_terrain.yaml widths: norms, first rows and sample outputs only
SEPT_SMALL = dict(S=22, traj=6, heightmap=30, A=11, amp=40, units=(96, 64, 48), task_units=(40, 24), disc_units=(32, 16), M=96, B=32, seed=31)
SEPT_FULL = dict(S=358, traj=20, heightmap=1024, A=32, amp=1960, units=(2048, 1024, 512), task_units=(512, 256), disc_units=(1024, 512),
                 M=64, B=32, seed=32)


def sept_fixture(d):
    """(state dict under the reference's parameter names without prefix, batch dict, checksum).  The batch holds RAW observations and the
    normaliser statistics they are normalised with (obs_mean / obs_var, amp_mean / amp_var)."""
    g = torch.Generator().manual_seed(d["seed"])
    sd = {}

    def lin(name, n_out, n_in, wscale=1.0, bscale=0.05):
        sd[name + ".weight"] = _uniform_pm1((n_out, n_in), g) * (wscale / n_in ** 0.5)
        sd[name + ".bias"] = _uniform_pm1((n_out,), g) * bscale

    def stack(name, n_in, units, wscale):
        for i, u in enumerate(units):
            lin(f"{name}.{2 * i}", u, n_in, wscale=wscale)
            n_in = u
        return n_in

    S, T, A = d["S"], d["traj"] + d["heightmap"], d["A"]
    E = stack("_task_mlp", T, d["task_units"], 2.0)
    for net, head, n_out in (("actor_mlp", "mu", A), ("critic_mlp", "value", 1)):
        n = stack(net, S + E, d["units"], 2.0)             # gain that keeps the SiLU stacks' activations O(1)
        lin(head, n_out, n, wscale=2.0, bscale=0.8)          # some |mu| past the soft bound: a non-zero bound loss
    n = stack("_disc_mlp", d["amp"], d["disc_units"], 1.5)
    lin("_disc_logits", 1, n)
    sd["sigma"] = torch.full((A,), -1.0)                   # pulse_z_terrain.yaml: fixed sigma, const_initializer -1
    M, B = d["M"], d["B"]
    b = dict(obs=_approx_normal((M, S + T), g) * 1.5 + 0.25, obs_mean=_uniform_pm1((S + T,), g) * 0.3, obs_var=1.0 + 0.5 * _uniform_pm1((S + T,), g),
             actions=_approx_normal((M, A), g) * 0.6, advantages=_approx_normal((M,), g), returns=_approx_normal((M,), g) * 0.5,
             amp_agent=_approx_normal((B, d["amp"]), g), amp_replay=_approx_normal((B, d["amp"]), g) * 1.2,
             amp_demo=_approx_normal((B, d["amp"]), g) * 0.8 + 0.2, amp_mean=_uniform_pm1((d["amp"],), g) * 0.2,
             amp_var=1.0 + 0.4 * _uniform_pm1((d["amp"],), g))
    chk = sum(float(v.double().sum()) for v in sd.values()) + sum(float(v.double().sum()) for v in b.values())
    return sd, b, chk


def normalise(x, mean, var):
    """RunningMeanStd.forward in eval mode (phc/utils/running_mean_std.py:69-95) with the given statistics."""
    return torch.clamp((x - mean.to(x.device, torch.float32)) / torch.sqrt(var.to(x.device, torch.float32) + 1e-5), -5.0, 5.0)
