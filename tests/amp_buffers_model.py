"""A numpy model of the device AMP rings (pulse_b200/csrc/amp_buffers.cu, include/pulse_b200.h) (TEST INFRASTRUCTURE): the reference's
ReplayBuffer bookkeeping (learning/replay_buffer.py) and `_store_replay_amp_obs` (amp_agent.py:1043-1057) with the device's draws in
place of torch.randperm / torch.bernoulli: the keyed Feistel permutation, the Philox keep mask and the subset permutation.  The ring
holds row ids, so what a store wrote and what a sample read can be compared with the device's index outputs and with the reference run
on the same draws (tests/golden/make_golden_amp_buffers.py)."""
import numpy as np

from tests.philox_ref import philox4x32_10, u01

PLANE_DEMO_CLIP, PLANE_DEMO_TIME, PLANE_REPLAY_KEEP, PLANE_REPLAY_SUBSET, PLANE_RING_PERM = 5, 6, 7, 8, 9
_M32 = 0xFFFFFFFF


def _fmix32(h: np.ndarray) -> np.ndarray:
    h = h ^ (h >> np.uint64(16))
    h = (h * np.uint64(0x85EBCA6B)) & np.uint64(_M32)
    h = h ^ (h >> np.uint64(13))
    h = (h * np.uint64(0xC2B2AE35)) & np.uint64(_M32)
    return h ^ (h >> np.uint64(16))


def feistel(seed: int, plane: int, counter: int, m: int, x) -> np.ndarray:
    """The device's keyed bijection of [0, m) applied to x (int array): four Feistel rounds on 2h bits, cycle-walked."""
    x = np.asarray(x, dtype=np.int64).copy()
    if m <= 1:
        return np.zeros_like(x)
    keys = [np.uint64(int(w[0])) for w in philox4x32_10(seed, [plane << 32], counter)]
    bits = 2
    while bits < 62 and (1 << bits) < m:
        bits += 1
    bits += bits & 1
    half = bits >> 1
    mask = np.uint64((1 << half) - 1)
    todo = np.ones(x.shape, dtype=bool)
    while todo.any():
        v = x[todo].astype(np.uint64)
        left, right = v >> np.uint64(half), v & mask
        for k in keys:
            f = _fmix32(((right * np.uint64(0x9E3779B1)) & np.uint64(_M32)) ^ k) & mask
            left, right = right, left ^ f
        x[todo] = ((left << np.uint64(half)) | right).astype(np.int64)
        todo = x >= m
    return x


def permutation(seed: int, plane: int, counter: int, m: int) -> np.ndarray:
    """perm[i] = the bijection's image of i: what the device uses in place of torch.randperm(m)."""
    return feistel(seed, plane, counter, m, np.arange(m))


def keep_mask(seed: int, draws: int, n: int, keep_prob: float) -> np.ndarray:
    """The Bernoulli(keep_prob) mask of a replay store: u01(word x of (seed, 7 * 2^32 + r, draws)) < keep_prob."""
    w = philox4x32_10(seed, [(PLANE_REPLAY_KEEP << 32) + r for r in range(n)], draws)[0]
    return u01(w) < np.float32(keep_prob)


class RingModel:
    """One ring: capacity rows of ids, the device counters (head, total_count, sample_head, perm_key, draws)."""

    def __init__(self, capacity: int, seed: int):
        self.cap, self.seed = int(capacity), int(seed)
        self.ids = np.full(self.cap, -1, dtype=np.int64)
        self.head = self.total = self.sample_head = self.perm_key = self.draws = 0

    def perm(self) -> np.ndarray:
        return permutation(self.seed, PLANE_RING_PERM, self.perm_key, self.cap)

    def _write(self, ids: np.ndarray) -> None:
        n = len(ids)
        assert n <= self.cap
        self.ids[(self.head + np.arange(n)) % self.cap] = ids
        self.head = (self.head + n) % self.cap
        self.total += n
        self.draws += 1

    def store(self, ids) -> None:
        """ReplayBuffer.store (the demo ring's fetches)."""
        self._write(np.asarray(ids, dtype=np.int64))

    def store_replay(self, ids, keep_prob: float) -> np.ndarray:
        """_store_replay_amp_obs: returns the source row (index into ids) of each stored row."""
        ids = np.asarray(ids, dtype=np.int64)
        rows = np.arange(len(ids))
        if self.total > self.cap:
            rows = rows[keep_mask(self.seed, self.draws, len(ids), keep_prob)]
        if len(rows) > self.cap:
            rows = rows[permutation(self.seed, PLANE_REPLAY_SUBSET, self.draws, len(rows))[:self.cap]]
        self._write(ids[rows])
        return rows

    def sample(self, n: int) -> np.ndarray:
        """ReplayBuffer.sample(n): the ring rows read, or None while the ring is empty (train_epoch then takes the agent's rows and
        the counters stay)."""
        if self.total == 0:
            return None
        idx = (self.sample_head + np.arange(n)) % self.cap
        r = self.perm()[idx]
        if self.total < self.cap:
            r = r % self.head
        self.sample_head += n
        if self.sample_head >= self.cap:
            self.sample_head = 0
            self.perm_key += 1
        return r

    def counters(self):
        return np.array([self.head, self.total, self.sample_head, self.perm_key, self.draws], dtype=np.int64)


# The scripted sequence: every branch of ReplayBuffer / _store_replay_amp_obs is crossed (see the fixture generator).
CAPACITY, SEED, KEEP_PROB = 64, 0x5EED, 0.9
SCRIPT = (("sample", 16),     # empty: the agent's rows
          ("store", 40),      # not full; no mask, no subset
          ("sample", 24),     # total < capacity: indices % head
          ("store", 40),      # head wraps
          ("sample", 48),     # full; sample_head reaches capacity: new permutation key
          ("store", 100),     # total > capacity: keep mask; more than capacity kept: subset
          ("store", 50),      # keep mask again, head wraps
          ("sample", 100))    # more than capacity in one sample: positions wrap, then a new key


def run_script(model: RingModel, keep_prob: float = KEEP_PROB):
    """Runs SCRIPT on `model`; returns per step (kind, rows, counters after) with rows = sampled ring rows (-1: agent rows) or the
    stored source rows, and the ring's ids after every step.  Stored batches carry ids 1000 * (step + 1) + row."""
    out = []
    for s, (kind, n) in enumerate(SCRIPT):
        if kind == "sample":
            r = model.sample(n)
            rows = np.full(n, -1, dtype=np.int64) if r is None else r
        else:
            rows = model.store_replay(1000 * (s + 1) + np.arange(n), keep_prob)
        out.append((kind, rows, model.counters(), model.ids.copy()))
    return out
