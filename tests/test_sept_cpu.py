"""oracle/sept_oracle.py (torch fp32 restatement of the amp_sept policy and its calc_gradients loss) against the reference-generated
tests/golden/sept.npz: (a) shrunk widths with every parameter gradient, (b) pulse_z_terrain.yaml widths."""
import pytest
import torch

from tests.helpers import load_npz
from tests.sept_fixture import SEPT_FULL, SEPT_SMALL, normalise, sept_fixture

TOL = 2e-6


def param_names(g, tag):
    """the reference network's trainable parameter names, in named_parameters() order"""
    return bytes(g[tag + "names"].numpy()).decode().split("\n")


def oracle_run(d, old_neglogp, device="cpu"):
    from oracle import sept_oracle as so
    sd, b, chk = sept_fixture(d)
    sd = {k: v.to(device).requires_grad_(k != "sigma") for k, v in sd.items()}
    b = {k: v.to(device) for k, v in b.items()}
    obs = normalise(b["obs"], b["obs_mean"], b["obs_var"])
    amp = [normalise(b[k], b["amp_mean"], b["amp_var"]) for k in ("amp_agent", "amp_replay", "amp_demo")]
    out = so.total_loss(sd, obs, b["actions"], old_neglogp.to(device), b["advantages"], b["returns"], amp=amp, self_obs_size=d["S"])
    names = [k for k in sd if k != "sigma"]
    grads = torch.autograd.grad(out["loss"], [sd[k] for k in names])
    return out, dict(zip(names, grads)), chk


def _close(a, b, tol=TOL):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert a.shape == b.shape, (a.shape, b.shape)
    err = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
    assert err <= tol, err


@pytest.mark.parametrize("tag,d", [("a_", SEPT_SMALL), ("b_", SEPT_FULL)])
def test_oracle_matches_reference_fixture(tag, d):
    g = load_npz("sept.npz")
    out, grads, chk = oracle_run(d, g[tag + "old_neglogp"])
    assert abs(chk - float(g[tag + "checksum"])) < 1e-9 * abs(chk), "regenerated fixture differs from the one the golden was made with"
    for k in ("a_loss", "c_loss", "b_loss", "disc_loss", "loss"):
        _close(out[k].detach(), g[tag + k])
    n = g[tag + "mu"].shape[0]
    _close(out["mu"].detach()[:n], g[tag + "mu"])
    _close(out["value"].detach()[:n], g[tag + "value"])
    names = param_names(g, tag)
    assert sorted(names) == sorted(grads), "the oracle's parameters are the reference network's trainable parameters"
    assert any(n.startswith("_task_mlp.") for n in names)
    for n in names:
        if tag == "a_":
            _close(grads[n], g[tag + "grad." + n])
        else:
            _close(grads[n].double().norm(), g[tag + "gnorm." + n], 1e-5)
            gr = grads[n]
            _close(gr.reshape(gr.shape[0], -1)[0] if gr.dim() > 1 else gr, g[tag + "grow0." + n], 1e-5)
