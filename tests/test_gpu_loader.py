"""Device-side MotionLib loader (SURVEY 8f-1) against the reference-generated tables (tests/golden/loader.npz): eight clips of
2 to 150 frames with the reference's heading randomisation.  Tolerances: rotations / positions 1e-5; velocities 2e-4 (gaussian of finite
differences); dof velocities 1e-3 -- the reference computes them from float32 local rotations with an acos near 1, so two
float32 implementations differ by ~2e-4 on slow joints.
"""
import pytest
import torch

from tests.helpers import load_npz

pytestmark = pytest.mark.gpu


def _fixture_clips(z):
    nf = z["num_frames"].tolist()
    clips, start = [], 0
    for i, n in enumerate(nf):
        a, b = start, start + n
        start = b
        clips.append({"pose_quat_global": z["in_pose_quat_global"][a:b].numpy(), "root_trans_offset": z["in_root_trans"][a:b],
                      "pose_aa": z["in_pose_aa"][a:b].numpy(), "fps": float(z["fps"][i])})
    return clips


def test_device_loader_matches_reference_tables_mixed_fps():
    """loader_fps.npz: the reference's tables for clips at 24 to 120 fps.  Velocities scale with the rate, so their tolerances scale with
    fps / 30 frame by frame; lengths and dt are the reference's float64 1 / fps rounded once."""
    from pulse_b200.motion_lib import MotionLibB200
    z = load_npz("loader_fps.npz")
    ml = MotionLibB200.from_clips(_fixture_clips(z), z["parents"].tolist(), z["local_translation"].numpy(), "cuda:0", headings=z["headings"].numpy())
    scale = torch.repeat_interleave(z["fps"].double() / 30.0, z["num_frames"]).reshape(-1, 1, 1)
    for k, t, scaled in (("gts", 1e-5, False), ("grs", 1e-6, False), ("lrs", 1e-6, False), ("gvs", 2e-4, True), ("gavs", 2e-4, True),
                         ("dvs", 1e-3, True)):
        got, want = getattr(ml, k).cpu().double(), z[k]
        tol = t * (scale if scaled else 1.0) + 1e-5 * want.abs()
        bad = (got - want).abs() > tol
        assert not bool(bad.any()), f"{k}: {int(bad.sum())} elements off, worst {float(((got - want).abs() / tol).max()):.3f} x tol"
    fps = z["fps"].tolist()
    nf = z["num_frames"].tolist()
    assert torch.equal(ml._motion_lengths.cpu(), torch.tensor([1.0 / f * (n - 1) for f, n in zip(fps, nf)], dtype=torch.float32))
    assert torch.equal(ml._motion_dt.cpu(), torch.tensor([1.0 / f for f in fps], dtype=torch.float32))


def test_device_loader_matches_reference_tables():
    from pulse_b200.motion_lib import MotionLibB200
    z = load_npz("loader.npz")
    nf = z["num_frames"].tolist()
    clips, start = [], 0
    for i, n in enumerate(nf):
        a, b = start, start + n
        start = b
        clips.append({"pose_quat_global": z["in_pose_quat_global"][a:b].numpy(), "root_trans_offset": z["in_root_trans"][a:b],
                      "pose_aa": z["in_pose_aa"][a:b].numpy(), "fps": float(z["fps"][i])})
    ml = MotionLibB200.from_clips(clips, z["parents"].tolist(), z["local_translation"].numpy(), "cuda:0", headings=z["headings"].numpy())
    tol = {"gts": 1e-5, "grs": 1e-6, "lrs": 1e-6, "gvs": 2e-4, "gavs": 2e-4, "dvs": 1e-3}
    for k, t in tol.items():
        torch.testing.assert_close(getattr(ml, k).cpu().double(), z[k], atol=t, rtol=1e-5, msg=lambda m, k=k: f"{k}: {m}")
    tables = load_npz("motionlib.npz")
    torch.testing.assert_close(ml._motion_lengths.cpu(), tables["lengths"], atol=0, rtol=0)
    assert torch.equal(ml.length_starts.cpu(), tables["length_starts"]) and torch.equal(ml._motion_num_frames.cpu(), tables["num_frames"])


def test_dataset_load_motions_reproduces_the_reference_tables():
    """`MotionDatasetB200.load_motions(random_sample=False)` = the reference's `load_motions` on the same clips (motionlib.npz was
    produced by exactly that call, make_golden.py): clip selection + heading protocol + device loader end to end."""
    from pulse_b200.motion_dataset import MotionDatasetB200
    z = load_npz("loader.npz")
    tables = load_npz("motionlib.npz")
    nf = z["num_frames"].tolist()
    clips, start = {}, 0
    for i, n in enumerate(nf):
        a, b = start, start + n
        start = b
        clips[f"clip_{i:02d}"] = {"pose_quat_global": z["in_pose_quat_global"][a:b].numpy(), "root_trans_offset": z["in_root_trans"][a:b],
                                  "pose_aa": z["in_pose_aa"][a:b].numpy(), "fps": float(z["fps"][i]), "beta": 0}
    ds = MotionDatasetB200(clips, z["parents"].tolist(), z["local_translation"].numpy(), device="cuda:0")
    ml = ds.load_motions(len(nf), random_sample=False)
    tol = {"gts": 1e-5, "grs": 1e-6, "lrs": 1e-6, "gvs": 2e-4, "gavs": 2e-4, "dvs": 1e-3}
    for k, t in tol.items():
        torch.testing.assert_close(getattr(ml, k).cpu(), tables[k], atol=t, rtol=1e-5, msg=lambda m, k=k: f"{k}: {m}")
    torch.testing.assert_close(ml._motion_aa.cpu(), tables["motion_aa"], atol=0, rtol=0)
