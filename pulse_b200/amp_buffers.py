"""The AMP demo and replay buffers of `AMPAgent` on the device (learning/replay_buffer.py `ReplayBuffer`; `_init_amp_demo_buf`,
`_update_amp_demos`, `_store_replay_amp_obs` and the buffer samples of `train_epoch`, phc/learning/amp_agent.py:476-484, :988-1057).
Every counter (head, total_count, sample_head, the permutation key) lives on the device, so no call synchronises with the host and
every call can be captured into a CUDA graph.  The draws are Philox / Feistel (include/pulse_b200.h) in place of torch.randperm and
torch.bernoulli; the bookkeeping is the reference's."""
import ctypes as C
import math
from typing import Optional

import torch

from . import _lib

# the AMP row widths per body layout: with the root height, without it (ampRootHeightObs)
AMP_WIDTHS = {"smpl": (196, 195), "smplx": (_lib.SMPLX_AMP_OBS, _lib.SMPLX_AMP_OBS_NO_HEIGHT)}
_DEMO_FETCH = {"smpl": "pulse_amp_demo_fetch", "smplx": "pulse_smplx_amp_demo_fetch"}


class AmpRing:
    """One ReplayBuffer of `capacity` AMP rows of `row_floats` floats, with its device counters."""

    def __init__(self, capacity: int, row_floats: int, seed: int, device):
        self.capacity, self.row_floats, self.device = int(capacity), int(row_floats), torch.device(device)
        self.rows = torch.zeros(self.capacity, self.row_floats, device=self.device)
        self.ctr = torch.zeros(_lib.RING_CTRS, dtype=torch.int64, device=self.device)
        self.seed = int(seed) & (2 ** 64 - 1)

    def desc(self) -> _lib.AmpRing:
        return _lib.AmpRing(rows=self.rows.data_ptr(), capacity=self.capacity, ctr=self.ctr.data_ptr(), seed=self.seed, row_floats=self.row_floats)

    def counters(self) -> torch.Tensor:
        """(head, total_count, sample_head, perm_key, draws) -- a device tensor view."""
        return self.ctr[:5]


class AmpBuffersB200:
    """The demo ring filled from the MotionLib and the replay ring of the policy's own AMP rows.

    `motion_lib`: the MotionLibB200 the demo rows come from; `sampling_cdf` its clip CDF (default: the MotionLib's).  `num_steps` x
    `amp_width` and `upright` are the env's AMP layout, `dt` its control step: a 24-body SMPL MotionLib takes 196 floats, or 195
    without the root height, upright or not; a 52-body SMPL-X one (PULSE-X, env_pulsex_amp.yaml) takes 466 or 465 and upright=False
    (`pulse_smplx_amp_demo_fetch`).  The sizes and the keep probability are the learning config's amp_obs_demo_buffer_size,
    amp_replay_buffer_size, amp_batch_size, amp_replay_keep_prob and amp_minibatch_size.  Memory: capacity * num_steps * amp_width * 4
    bytes per ring (1.57 GB for 200 000 rows of 10 x 196 floats, 3.72 GB for 200 000 rows of 10 x 465)."""

    def __init__(self, motion_lib, *, num_steps: int = 10, amp_width: int = 196, upright: bool = True, dt: float = float(torch.tensor(1.0 / 60.0, dtype=torch.float32) * 2),
                 demo_buffer_size: int = 200000, replay_buffer_size: int = 200000, batch_size: int = 512, keep_prob: float = 0.01,
                 minibatch_size: int = 4096, seed: int = 0, sampling_cdf: Optional[torch.Tensor] = None):
        self.smplx = bool(getattr(motion_lib, "smplx", False))
        self.layout = "smplx" if self.smplx else "smpl"
        widths = AMP_WIDTHS[self.layout]
        if amp_width not in widths:
            raise _lib.PulseError(f"amp_width {amp_width}: the {self.layout} AMP rows are {widths[0]} floats, or {widths[1]} without the root "
                                  f"height")
        if self.smplx and upright:
            raise _lib.PulseError("the SMPL-X AMP rows take upright=False (env_pulsex_amp.yaml: has_upright_start False)")
        if not 1 <= batch_size <= demo_buffer_size:
            raise _lib.PulseError(f"amp_batch_size {batch_size} must lie in [1, amp_obs_demo_buffer_size]")
        self.motion_lib, self.device = motion_lib, motion_lib._device
        self.num_steps, self.amp_width, self.upright, self.dt = int(num_steps), int(amp_width), bool(upright), float(dt)
        self.row_floats = self.num_steps * self.amp_width
        self.batch_size, self.keep_prob, self.minibatch_size = int(batch_size), float(keep_prob), int(minibatch_size)
        base = (int(seed) * 0x9E3779B97F4A7C15 + 0x452821E638D01377) & (2 ** 64 - 1)
        self.demo = AmpRing(demo_buffer_size, self.row_floats, base, self.device)
        self.replay = AmpRing(replay_buffer_size, self.row_floats, base ^ 0xBE5466CF34E90C6C, self.device)
        self._cdf = sampling_cdf
        self.lib = _lib.load()
        self._kept = None
        self.demo_filled = False

    def _stream(self):
        return _lib.current_stream(self.device)

    def cdf(self) -> torch.Tensor:
        return self._cdf if self._cdf is not None else self.motion_lib.sampling_cdf()

    # ------------------------------------------------------------------ demo ring
    def fetch_demos(self, num_samples: Optional[int] = None, motion_ids_out: Optional[torch.Tensor] = None,
                    times_out: Optional[torch.Tensor] = None) -> None:
        """`_amp_obs_demo_buffer.store(fetch_amp_obs_demo(num_samples))` in one call (`pulse_amp_demo_fetch`, `pulse_smplx_amp_demo_fetch`
        for SMPL-X); the optional outputs receive the drawn clips and start times."""
        n = self.batch_size if num_samples is None else int(num_samples)
        a = _lib.AmpDemoArgs(ring=self.demo.desc(), sampling_cdf=self.cdf().data_ptr(), num_samples=n, num_steps=self.num_steps,
                             amp_width=self.amp_width, upright=int(self.upright), dt=self.dt, motion_ids_out=_lib.ptr(motion_ids_out),
                             times_out=_lib.ptr(times_out))
        fn = _DEMO_FETCH[self.layout]
        handle = self.motion_lib.smplx_handle if self.smplx else self.motion_lib.handle
        with torch.cuda.device(self.device):
            _lib.check(getattr(self.lib, fn)(handle, C.byref(a), self._stream()), fn)

    def init_demo(self) -> None:
        """`_init_amp_demo_buf`: ceil(buffer_size / amp_batch_size) fetches of amp_batch_size rows, wrapping as the ring does."""
        for _ in range(math.ceil(self.demo.capacity / self.batch_size)):
            self.fetch_demos()
        self.demo_filled = True

    def update_demos(self) -> None:
        """`_update_amp_demos`: one fetch of amp_batch_size rows, after `init_demo` if it has not run yet (the reference fills the demo
        buffer when the agent is built, before the first epoch)."""
        if not self.demo_filled:
            self.init_demo()
        self.fetch_demos()

    # ------------------------------------------------------------------ samples
    def sample(self, ring: AmpRing, n: int, block: int, out: torch.Tensor, fallback: Optional[torch.Tensor] = None,
               ring_rows_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`ring.sample(n)` restricted to the rows the update reads: the first amp_minibatch_size rows of every `block`-row minibatch,
        into `out` [n / block * take, row_floats]; sample_head still moves by n.  `fallback` [n, row_floats]: the rows taken while the
        ring is empty (the agent's own rows, train_epoch's `amp_obs_replay = amp_obs`)."""
        take = min(self.minibatch_size, int(block))
        if out.shape != (n // block * take, self.row_floats) or not out.is_contiguous():
            raise _lib.PulseError(f"out must be contiguous [{n // block * take}, {self.row_floats}]")
        if fallback is not None and (fallback.shape[0] < n or not fallback.is_contiguous() or fallback.numel() != fallback.shape[0] * self.row_floats):
            raise _lib.PulseError(f"fallback must be contiguous [{n}, {self.row_floats}]")
        a = _lib.AmpSampleArgs(ring=ring.desc(), n=int(n), block=int(block), take=take, fallback=_lib.ptr(fallback), out=out.data_ptr(),
                               ring_rows_out=_lib.ptr(ring_rows_out))
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_amp_ring_sample(C.byref(a), self._stream()), "pulse_amp_ring_sample")
        return out

    # ------------------------------------------------------------------ replay ring
    def store_replay(self, amp_obs: torch.Tensor, src_rows_out: Optional[torch.Tensor] = None) -> None:
        """`_store_replay_amp_obs(amp_obs)` (`pulse_amp_replay_store`) of the horizon's rows [rows, row_floats]."""
        rows = int(amp_obs.shape[0])
        if not amp_obs.is_contiguous() or amp_obs.numel() != rows * self.row_floats or amp_obs.dtype != torch.float32:
            raise _lib.PulseError(f"amp_obs must be contiguous float32 [rows, {self.row_floats}]")
        if self._kept is None or self._kept.shape[0] < rows:
            self._kept = torch.zeros(rows, dtype=torch.int32, device=self.device)
        a = _lib.AmpStoreArgs(ring=self.replay.desc(), src=amp_obs.data_ptr(), num_rows=rows, keep_prob=self.keep_prob,
                              kept=self._kept.data_ptr(), src_rows_out=_lib.ptr(src_rows_out))
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pulse_amp_replay_store(C.byref(a), self._stream()), "pulse_amp_replay_store")
