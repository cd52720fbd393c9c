"""The AMP replay ring on the device (`pulse_b200.amp_buffers`, csrc/amp_buffers.cu): its stored and sampled rows and its counters word
for word against the numpy model (tests/amp_buffers_model.py, itself checked against the reference's ReplayBuffer and
_store_replay_amp_obs), whose keep mask is drawn with tests/philox_ref.py.  The demo fetch and the drivers: test_gpu_latent_amp.py."""
import numpy as np
import pytest
import torch

from tests import amp_buffers_model as M
from tests.test_gpu_ztask_rollout import motion  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_replay_ring_matches_model(motion):
    from pulse_b200.amp_buffers import AmpRing, AmpBuffersB200
    ml, _ = motion
    bufs = AmpBuffersB200(ml, num_steps=2, amp_width=196, demo_buffer_size=8, replay_buffer_size=M.CAPACITY, batch_size=4,
                          keep_prob=M.KEEP_PROB, minibatch_size=10 ** 9)
    ring = bufs.replay = AmpRing(M.CAPACITY, 392, M.SEED, DEV)
    model = M.RingModel(M.CAPACITY, M.SEED)
    for s, (kind, n) in enumerate(M.SCRIPT):
        ids = 1000 * (s + 1) + torch.arange(n, device=DEV, dtype=torch.float32)
        rows = ids[:, None].expand(n, 392).contiguous()
        if kind == "sample":
            out = torch.empty(n, 392, device=DEV)
            got = torch.empty(n, dtype=torch.int64, device=DEV)
            bufs.sample(ring, n, n, out, fallback=rows, ring_rows_out=got)
            want = model.sample(n)
            want = np.full(n, -1) if want is None else want
            np.testing.assert_array_equal(got.cpu().numpy(), want, err_msg=f"step {s}")
            want_rows = rows[:, 0].cpu().numpy() if (want < 0).all() else model.ids[want]
            np.testing.assert_array_equal(out[:, 0].cpu().numpy().astype(np.int64), want_rows)
        else:
            src = torch.empty(min(n, M.CAPACITY), dtype=torch.int64, device=DEV)
            bufs.store_replay(rows, src_rows_out=src)
            want = model.store_replay(ids.cpu().numpy().astype(np.int64), M.KEEP_PROB)
            got = src.cpu().numpy()
            np.testing.assert_array_equal(got[:len(want)], want, err_msg=f"step {s}")
            assert (got[len(want):] == -1).all()
        np.testing.assert_array_equal(ring.counters().cpu().numpy(), model.counters(), err_msg=f"step {s}")
        stored = ring.rows[:, 0].cpu().numpy().astype(np.int64)
        np.testing.assert_array_equal(np.where(model.ids < 0, 0, model.ids), stored)
        assert torch.equal(ring.rows, ring.rows[:, :1].expand_as(ring.rows))


def test_sample_gathers_first_rows_of_each_minibatch(motion):
    from pulse_b200.amp_buffers import AmpRing, AmpBuffersB200
    ml, _ = motion
    bufs = AmpBuffersB200(ml, num_steps=1, amp_width=196, demo_buffer_size=8, replay_buffer_size=50, batch_size=4, minibatch_size=3)
    ring = AmpRing(50, 196, 77, DEV)
    ring.rows.copy_(torch.arange(50, device=DEV, dtype=torch.float32)[:, None].expand(50, 196))
    ring.ctr[1] = 60                     # full
    model = M.RingModel(50, 77)
    model.total, model.ids = 60, np.arange(50)
    out = torch.empty(4 * 3, 196, device=DEV)
    idx = torch.empty(12, dtype=torch.int64, device=DEV)
    bufs.sample(ring, 40, 10, out, ring_rows_out=idx)
    full = model.sample(40)
    want = np.concatenate([full[b * 10:b * 10 + 3] for b in range(4)])
    np.testing.assert_array_equal(idx.cpu().numpy(), want)
    np.testing.assert_array_equal(out[:, 5].cpu().numpy(), want.astype(np.float32))
    assert int(ring.ctr[2]) == 40
