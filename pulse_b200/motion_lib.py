"""Device-resident MotionLib: host-side mirror of the query API of
`phc.utils.motion_lib_base.MotionLibBase` / `motion_lib_smpl.MotionLibSMPL` (reference), backed by
the packed per-frame records and the CUDA query kernel of libpulse_b200.so.

Same method names, argument meaning and return keys as the reference:
  get_motion_state(motion_ids, motion_times, offset=None)   motion_lib_base.py:434-517
  get_root_pos_smpl(motion_ids, motion_times)               motion_lib_base.py:519-544
  sample_time_interval(motion_ids, truncate_time=None)      motion_lib_base.py:411-420
  sample_time / get_motion_length / num_motions / get_motion_num_steps
The clip loader (load_motions: FK, heading randomisation, velocity filters) stays with the
reference for now (SURVEY.md 8f-1): build this object from the tables it produced with
`MotionLibB200.from_reference(motion_lib)` or from raw tables with `from_tables(...)`.  `from_clips(...)` is the
device-side loader (SURVEY 8f-1): parity green against the reference's tables (tests/test_gpu_loader.py).

The tables' body count chooses the humanoid: 24 bodies is SMPL, 52 the SMPL-X humanoid of PULSE-X (smplx_humanoid.xml, 153 dofs),
whose records (PULSE_SMPLX_FRAME_REC / PULSE_SMPLX_AUX_REC) and queries are the `pulse_smplx_*` entry points.  `from_reference` adopts a
loaded SMPL-X MotionLib as it adopts an SMPL one; `from_clips` (the forward-kinematics loader) is SMPL only.
"""
import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib

FRAME_REC = 312
AUX_REC = 240
SMPLX_FRAME_REC, SMPLX_AUX_REC = 676, 364
_TABLE_KEYS = ("gts", "grs", "lrs", "gvs", "gavs", "dvs")


class MotionLibB200:
    def __init__(self, tables: Dict[str, torch.Tensor], device=None):
        """tables: gts grs lrs gvs gavs dvs [motion_aa] lengths num_frames dt length_starts
        [fps motion_bodies motion_limb_weights] with the reference's shapes (motion_lib_base.py:287-316)."""
        lib = _lib.load()
        dev = torch.device(device) if device is not None else tables["gts"].device
        if dev.type != "cuda":
            raise _lib.PulseError("MotionLibB200 needs a CUDA device (no CPU fallback)")
        self._device = dev
        f32 = lambda x: x.to(dev, torch.float32).contiguous()
        i64 = lambda x: x.to(dev, torch.int64).contiguous()
        self.gts, self.grs, self.lrs = f32(tables["gts"]), f32(tables["grs"]), f32(tables["lrs"])
        self.gvs, self.gavs, self.dvs = f32(tables["gvs"]), f32(tables["gavs"]), f32(tables["dvs"])
        F, B = self.gts.shape[0], self.gts.shape[1]
        if (B not in (24, _lib.SMPLX_BODIES) or self.gts.shape[2:] != (3,) or self.grs.shape != (F, B, 4) or self.lrs.shape != (F, B, 4)
                or self.dvs.shape != (F, B - 1, 3)):
            raise _lib.PulseError(f"unexpected table shapes {tuple(self.gts.shape)} {tuple(self.grs.shape)} {tuple(self.dvs.shape)}: "
                                  "24 (SMPL) or 52 (SMPL-X) bodies")
        self.smplx = B == _lib.SMPLX_BODIES
        self._motion_aa = f32(tables["motion_aa"]) if tables.get("motion_aa") is not None else torch.zeros(F, 3 * B, device=dev)
        self._motion_lengths = f32(tables["lengths"])
        self._motion_num_frames = i64(tables["num_frames"])
        self._motion_dt = f32(tables["dt"])
        self.length_starts = i64(tables["length_starts"])
        M = self._motion_lengths.shape[0]
        self._motion_fps = f32(tables["fps"]) if tables.get("fps") is not None else 1.0 / self._motion_dt
        self._motion_bodies = f32(tables["motion_bodies"]) if tables.get("motion_bodies") is not None else torch.zeros(M, 17, device=dev)
        self._motion_limb_weights = (f32(tables["motion_limb_weights"]) if tables.get("motion_limb_weights") is not None
                                     else torch.zeros(M, 10, device=dev))
        self._num_motions = M
        self.num_bodies = B
        self.motion_ids = torch.arange(M, dtype=torch.long, device=dev)
        self._sampling_batch_prob = torch.full((M,), 1.0 / M, device=dev)
        self._time_step = torch.tensor(1 / 30, dtype=torch.float32, device=dev)  # cached: no H2D copy inside CUDA-graph capture

        handle = C.c_void_p()
        self._lib = lib
        if self.smplx:
            self._pack_smplx(F, M, handle)
            self._handle = handle
            return
        # packed records (layout: include/pulse_b200.h PULSE_FRAME_REC / PULSE_AUX_REC)
        self.frame_rec = torch.empty(F, FRAME_REC, device=dev, dtype=torch.float32)
        self.aux_rec = torch.empty(F, AUX_REC, device=dev, dtype=torch.float32)
        desc = _lib.MotionLibDesc(
            gts=self.gts.data_ptr(), grs=self.grs.data_ptr(), lrs=self.lrs.data_ptr(), gvs=self.gvs.data_ptr(),
            gavs=self.gavs.data_ptr(), dvs=self.dvs.data_ptr(), motion_aa=self._motion_aa.data_ptr(),
            lengths=self._motion_lengths.data_ptr(), dt=self._motion_dt.data_ptr(),
            num_frames=self._motion_num_frames.data_ptr(), length_starts=self.length_starts.data_ptr(),
            total_frames=F, num_motions=M, frame_rec=self.frame_rec.data_ptr(), aux_rec=self.aux_rec.data_ptr())
        with torch.cuda.device(dev):
            _lib.check(lib.pulse_motionlib_create(C.byref(desc), _lib.current_stream(dev), C.byref(handle)), "pulse_motionlib_create")
        self._handle = handle

    def _pack_smplx(self, F: int, M: int, handle) -> None:
        """The SMPL-X records (layout: include/pulse_b200.h PULSE_SMPLX_FRAME_REC / PULSE_SMPLX_AUX_REC) and their handle."""
        dev = self._device
        self.frame_rec = torch.empty(F, SMPLX_FRAME_REC, device=dev, dtype=torch.float32)
        self.aux_rec = torch.empty(F, SMPLX_AUX_REC, device=dev, dtype=torch.float32)
        desc = _lib.SmplxMotionLibDesc(
            gts=self.gts.data_ptr(), grs=self.grs.data_ptr(), lrs=self.lrs.data_ptr(), gvs=self.gvs.data_ptr(), gavs=self.gavs.data_ptr(),
            dvs=self.dvs.data_ptr(), lengths=self._motion_lengths.data_ptr(), dt=self._motion_dt.data_ptr(),
            num_frames=self._motion_num_frames.data_ptr(), length_starts=self.length_starts.data_ptr(), total_frames=F, num_motions=M,
            frame_rec=self.frame_rec.data_ptr(), aux_rec=self.aux_rec.data_ptr())
        with torch.cuda.device(dev):
            _lib.check(self._lib.pulse_smplx_motionlib_create(C.byref(desc), _lib.current_stream(dev), C.byref(handle)),
                       "pulse_smplx_motionlib_create")

    # ------------------------------------------------------------------ constructors
    @classmethod
    def from_tables(cls, tables, device=None):
        return cls(dict(tables), device=device)

    @classmethod
    def from_reference(cls, ref_lib, device=None):
        """Adopt the tables a loaded reference MotionLibSMPL holds (after load_motions), SMPL or SMPL-X."""
        t = {k: getattr(ref_lib, k) for k in _TABLE_KEYS}
        t.update(motion_aa=ref_lib._motion_aa, lengths=ref_lib._motion_lengths, num_frames=ref_lib._motion_num_frames,
                 dt=ref_lib._motion_dt, length_starts=ref_lib.length_starts, fps=ref_lib._motion_fps,
                 motion_bodies=ref_lib._motion_bodies, motion_limb_weights=ref_lib._motion_limb_weights)
        return cls(t, device=device)

    @classmethod
    def from_clips(cls, clips, parents, local_translation, device, headings=None):
        """Device-side loader (SURVEY 8f-1): build the tables ON THE DEVICE from
        clips in the on-disk schema (`pose_quat_global` f64 [T,24,4], `root_trans_offset` f64 [T,3], `pose_aa` [T,72], `fps`;
        convert_amass_isaac.py:127-136) instead of MotionLibBase.load_motions' per-frame Python loops
        (motion_lib_base.py:179-323).  `headings`: the per-clip heading angles the reference draws with
        `np.pi * (2 * np.random.random() - 1)` (motion_lib_smpl.py:134-135), or None for the im_eval / test path."""
        import numpy as np
        lib = _lib.load()
        dev = torch.device(device)
        nf = [int(np.asarray(c["pose_quat_global"]).shape[0]) for c in clips]
        M, F = len(clips), int(sum(nf))
        f64 = lambda arrs: torch.from_numpy(np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.float64) for a in arrs], axis=0))).to(dev)
        quat = f64([c["pose_quat_global"] for c in clips])
        trans = f64([c["root_trans_offset"].numpy() if torch.is_tensor(c["root_trans_offset"]) else c["root_trans_offset"] for c in clips])
        starts = torch.tensor(np.concatenate([[0], np.cumsum(nf)]), dtype=torch.int64, device=dev)
        frame_clip = torch.repeat_interleave(torch.arange(M, dtype=torch.int32, device=dev), torch.tensor(nf, device=dev))
        fps = torch.tensor([float(c.get("fps", 30)) for c in clips], dtype=torch.float32, device=dev)
        hd = torch.as_tensor(np.asarray(headings, dtype=np.float64)).to(dev) if headings is not None else None
        par = torch.as_tensor(np.asarray(parents, dtype=np.int32)).to(dev)
        loc = torch.as_tensor(np.asarray(local_translation, dtype=np.float32)).to(dev).contiguous()
        z = lambda *shape: torch.zeros(*shape, device=dev, dtype=torch.float32)
        t = {"gts": z(F, 24, 3), "grs": z(F, 24, 4), "lrs": z(F, 24, 4), "gvs": z(F, 24, 3), "gavs": z(F, 24, 3), "dvs": z(F, 23, 3)}
        tmp_v, tmp_w = z(F, 24, 3), z(F, 24, 3)
        a = _lib.LoaderArgs(pose_quat_global=quat.data_ptr(), root_trans=trans.data_ptr(), frame_clip=frame_clip.data_ptr(),
                            clip_start=starts.data_ptr(), fps=fps.data_ptr(), headings=_lib.ptr(hd), parents=par.data_ptr(),
                            local_translation=loc.data_ptr(), total_frames=F, num_clips=M, gts=t["gts"].data_ptr(), grs=t["grs"].data_ptr(),
                            lrs=t["lrs"].data_ptr(), gvs=t["gvs"].data_ptr(), gavs=t["gavs"].data_ptr(), dvs=t["dvs"].data_ptr(),
                            tmp_vel=tmp_v.data_ptr(), tmp_ang=tmp_w.data_ptr())
        with torch.cuda.device(dev):
            _lib.check(lib.pulse_motionlib_load_clips(C.byref(a), _lib.current_stream(dev)), "pulse_motionlib_load_clips")
        nf_t = torch.tensor(nf, dtype=torch.int64, device=dev)
        fps64 = [float(c.get("fps", 30)) for c in clips]
        t.update(motion_aa=torch.from_numpy(np.concatenate([np.asarray(c["pose_aa"]).reshape(-1, 72) for c in clips])).float(),
                 lengths=torch.tensor([1.0 / f * (n - 1) for f, n in zip(fps64, nf)], dtype=torch.float32),   # motion_lib_base.py:262-263
                 num_frames=nf_t, dt=torch.tensor([1.0 / f for f in fps64], dtype=torch.float32), length_starts=starts[:-1].clone(), fps=fps)
        return cls(t, device=dev)

    def __del__(self):
        h = getattr(self, "_handle", None)
        if h is not None and h.value:
            (self._lib.pulse_smplx_motionlib_destroy if self.smplx else self._lib.pulse_motionlib_destroy)(h)
            self._handle = None

    @property
    def handle(self):
        """The SMPL handle (`pulse_motionlib_t*`) every SMPL entry point takes; refused for SMPL-X tables, whose handle is another type."""
        if self.smplx:
            raise _lib.PulseError("this MotionLibB200 holds 52-body SMPL-X tables: the SMPL entry points cannot take it (smplx_handle is its "
                                  "handle, for the PULSE-X speed task's reset)")
        return self._handle

    @property
    def smplx_handle(self):
        """The SMPL-X handle (`pulse_smplx_motionlib_t*`) of 52-body tables; refused for SMPL tables."""
        if not self.smplx:
            raise _lib.PulseError("this MotionLibB200 holds 24-body SMPL tables: it has no SMPL-X handle")
        return self._handle

    # ------------------------------------------------------------------ reference API
    def num_motions(self):
        return self._num_motions

    def get_total_length(self):
        return sum(self._motion_lengths)

    def get_motion_length(self, motion_ids=None):
        return self._motion_lengths if motion_ids is None else self._motion_lengths[motion_ids]

    def get_motion_num_steps(self, motion_ids=None):
        nf = self._motion_num_frames if motion_ids is None else self._motion_num_frames[motion_ids]
        fps = self._motion_fps if motion_ids is None else self._motion_fps[motion_ids]
        return (nf * 30 / fps).int()

    def sample_motions(self, n):
        return torch.multinomial(self._sampling_batch_prob, num_samples=n, replacement=True).to(self._device)

    def sampling_cdf(self) -> torch.Tensor:
        """Inclusive fp32 prefix sum of `_sampling_batch_prob` on the device: the kernels draw clips by an inverse-CDF search of it.
        Rebuilt whenever `_sampling_batch_prob` is replaced or changed in place (the tensor's version counter), without reading it."""
        p = self._sampling_batch_prob
        if getattr(self, "_cdf_src", None) is not p or self._cdf_version != p._version:
            self._cdf = torch.cumsum(p.to(self._device, torch.float32), 0).contiguous()
            self._cdf_src, self._cdf_version = p, p._version
        return self._cdf

    def sample_time(self, motion_ids, truncate_time=None):
        phase = torch.rand(motion_ids.shape, device=self._device)
        motion_len = self._motion_lengths[motion_ids]
        if truncate_time is not None:
            assert truncate_time >= 0.0
            motion_len = motion_len - truncate_time
        return phase * motion_len

    def sample_time_interval(self, motion_ids, truncate_time=None, phase: Optional[torch.Tensor] = None):
        """motion_lib_base.py:411-420.  `phase` lets a test inject the uniform draw.  The division by
        the python scalar 1/30 follows the reference's CPU form (true fp32 division), not the
        multiply-by-reciprocal PyTorch-CUDA would use for tensor/scalar."""
        if phase is None:
            phase = torch.rand(motion_ids.shape, device=self._device)
        motion_len = self._motion_lengths[motion_ids]
        if truncate_time is not None:
            assert truncate_time >= 0.0
            motion_len = motion_len - truncate_time
        step = self._time_step
        return torch.div(phase * motion_len, step).long() * step

    def _query(self, motion_ids, motion_times, offset, want_full=True, diagnostics=False):
        n = int(motion_ids.shape[0])
        dev = self._device
        ids = motion_ids.to(dev, torch.int64).contiguous()
        times = motion_times.to(dev, torch.float32).contiguous()
        off = offset.to(dev, torch.float32).contiguous() if offset is not None else None
        mk = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        if self.smplx:
            return self._query_smplx(n, ids, times, off, want_full, diagnostics, mk), ids
        out = {"root_pos": mk(n, 3)}
        if want_full:
            out.update(root_rot=mk(n, 4), dof_pos=mk(n, 69), root_vel=mk(n, 3), root_ang_vel=mk(n, 3), dof_vel=mk(n, 69),
                       motion_aa=mk(n, 72), rg_pos=mk(n, 24, 3), rb_rot=mk(n, 24, 4), body_vel=mk(n, 24, 3),
                       body_ang_vel=mk(n, 24, 3))
        if diagnostics:
            out.update(frame_idx0=torch.empty(n, device=dev, dtype=torch.int64), frame_idx1=torch.empty(n, device=dev, dtype=torch.int64),
                       blend=mk(n))
        q = _lib.MotionQuery(motion_ids=ids.data_ptr(), motion_times=times.data_ptr(),
                             offset=off.data_ptr() if off is not None else None)
        for k, v in out.items():
            setattr(q, k, v.data_ptr())
        if n > 0:
            with torch.cuda.device(dev):
                _lib.check(self._lib.pulse_motion_state(self._handle, C.byref(q), n, _lib.current_stream(dev)), "pulse_motion_state")
        return out, ids

    def _query_smplx(self, n, ids, times, off, want_full, diagnostics, mk):
        if diagnostics:
            raise _lib.PulseError("the SMPL-X query has no frame diagnostics")
        B, D, dev = self.num_bodies, _lib.SMPLX_DOF, self._device
        out = {"root_pos": mk(n, 3)}
        if want_full:
            out.update(root_rot=mk(n, 4), dof_pos=mk(n, D), root_vel=mk(n, 3), root_ang_vel=mk(n, 3), dof_vel=mk(n, D), rg_pos=mk(n, B, 3),
                       rb_rot=mk(n, B, 4), body_vel=mk(n, B, 3), body_ang_vel=mk(n, B, 3))
        q = _lib.SmplxMotionQuery(motion_ids=ids.data_ptr(), motion_times=times.data_ptr(), offset=off.data_ptr() if off is not None else None)
        for k, v in out.items():
            setattr(q, k, v.data_ptr())
        if n > 0:
            with torch.cuda.device(dev):
                _lib.check(self._lib.pulse_smplx_motion_state(self._handle, C.byref(q), n, _lib.current_stream(dev)), "pulse_smplx_motion_state")
        return out

    def get_motion_state(self, motion_ids, motion_times, offset=None, diagnostics=False):
        out, ids = self._query(motion_ids, motion_times, offset, want_full=True, diagnostics=diagnostics)
        out["motion_bodies"] = self._motion_bodies[ids]
        out["motion_limb_weights"] = self._motion_limb_weights[ids]
        return out

    def get_root_pos_smpl(self, motion_ids, motion_times):
        out, _ = self._query(motion_ids, motion_times, None, want_full=False)
        return {"root_pos": out["root_pos"]}
