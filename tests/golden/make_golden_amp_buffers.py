"""Fixture for the AMP replay ring: the UNMODIFIED reference's `ReplayBuffer` (learning/replay_buffer.py) and
`AMPAgent._store_replay_amp_obs` (amp_agent.py:1043-1057) run through `tests.amp_buffers_model.SCRIPT`, with the train_epoch branch
`amp_obs_replay = amp_obs` while the buffer is empty (amp_agent.py:481-484).

  * `torch.randperm` and `torch.bernoulli` are wrapped to return the device's draws from the numpy model: randperm(capacity) is the
    sampling permutation of the next key (0 in the constructor, then one per `_reset_sample_idx`), randperm(m) for m != capacity the
    store's subset permutation, bernoulli the keep mask.  Everything else is the reference's own bookkeeping.
  * Stored rows carry their id, so the sampled rows and the buffer contents show what the reference read and wrote.

  python tests/golden/make_golden_amp_buffers.py     (needs the reference tree; writes tests/golden/amp_buffers.npz)
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def main():
    from oracle.refshim.load_reference import load_learning
    from tests import amp_buffers_model as M
    lrn = load_learning()
    cap, seed, p = M.CAPACITY, M.SEED, M.KEEP_PROB
    state = {"perm_key": 0, "draws": 0}
    real_randperm, real_bernoulli = torch.randperm, torch.bernoulli

    def randperm(n, *a, **k):
        if n == cap:
            perm = M.permutation(seed, M.PLANE_RING_PERM, state["perm_key"], cap)
            state["perm_key"] += 1
        else:
            perm = M.permutation(seed, M.PLANE_REPLAY_SUBSET, state["draws"], n)
        return torch.from_numpy(perm)

    def bernoulli(probs, *a, **k):
        return torch.from_numpy(M.keep_mask(seed, state["draws"], probs.shape[0], p).astype(np.float64)).to(probs.dtype)

    torch.randperm, torch.bernoulli = randperm, bernoulli
    try:
        buf = lrn.replay_buffer.ReplayBuffer(cap, "cpu")
        agent = types.SimpleNamespace(_amp_replay_buffer=buf, _amp_replay_keep_prob=p, ppo_device="cpu")
        out = {}
        for s, (kind, n) in enumerate(M.SCRIPT):
            if kind == "sample":
                if buf.get_total_count() == 0:
                    ids = np.full(n, -1)
                else:
                    ids = buf.sample(n)["amp_obs"][:, 0].numpy().astype(np.int64)
                out[f"s{s}_ids"] = ids
            else:
                rows = torch.arange(n, dtype=torch.float64)[:, None] + 1000 * (s + 1)
                lrn.amp_agent.AMPAgent._store_replay_amp_obs(agent, rows.float())
                state["draws"] += 1
            out[f"s{s}_counters"] = np.array([buf._head, buf._total_count, buf._sample_head, state["perm_key"] - 1, state["draws"]], dtype=np.int64)
            out[f"s{s}_buffer"] = buf._data_buf["amp_obs"][:, 0].numpy().astype(np.int64) if buf._data_buf is not None else np.zeros(cap, np.int64)
    finally:
        torch.randperm, torch.bernoulli = real_randperm, real_bernoulli
    np.savez_compressed(os.path.join(HERE, "amp_buffers.npz"), **out)
    print("wrote", os.path.join(HERE, "amp_buffers.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
