"""SURVEY 8f-4: the oracle's restatement of every compute_imitation_observations* variant against fixtures written by the UNMODIFIED
reference (tests/golden/make_golden_obs_versions.py)."""
import importlib.util
import os

import numpy as np
import torch

from oracle import pulse_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_obs_versions", os.path.join(HERE, "golden", "make_golden_obs_versions.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def oracle_obs(version, track, T, upright, body_state, rp, rr, rv, rw, dof_pos, ref_dof_pos):
    tr = torch.tensor(track)
    kw = {}
    if version == 2:
        kw = dict(dof_pos=dof_pos.reshape(-1, 23, 3)[:, tr[1:] - 1], ref_dof_pos=ref_dof_pos.reshape(-1, 23, 3)[:, tr[1:] - 1])
    return po.imitation_obs(version, body_state[:, 0, 0:3], body_state[:, 0, 3:7], body_state[:, tr, 0:3], body_state[:, tr, 3:7],
                            body_state[:, tr, 7:10], body_state[:, tr, 10:13], rp[:, tr], rr[:, tr], rv[:, tr], rw[:, tr], T, upright, **kw)


def test_oracle_matches_reference_fixture():
    m = _gen()
    z = np.load(os.path.join(HERE, "golden", "obs_versions.npz"))
    N = int(z["num_envs"])
    for k, (tag, version, track, T, upright) in enumerate(m.CASES):
        got = oracle_obs(version, track, T, upright, *m.inputs(N, T, 100 + k))
        ref = torch.from_numpy(z[tag])
        assert got.shape == ref.shape, tag
        torch.testing.assert_close(got, ref, atol=3e-6, rtol=3e-6, msg=lambda s, tag=tag: f"{tag}: {s}")
