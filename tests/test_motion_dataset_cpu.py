"""Host-side MotionLib dataset logic (pulse_b200/motion_dataset.py) without a GPU: clip selection, heading draws and the PMCP
sampling-weight updates against fixtures written by the reference's own methods."""
import numpy as np
import torch

from tests.helpers import load_npz


def _dataset(n=6):
    from pulse_b200.motion_dataset import MotionDatasetB200
    clips = {f"clip_{i:02d}": {"pose_quat_global": np.zeros((5 + i, 24, 4)), "pose_aa": np.zeros((5 + i, 72)),
                               "root_trans_offset": torch.zeros(5 + i, 3, dtype=torch.float64), "fps": 30.0} for i in range(n)}
    return MotionDatasetB200(clips, [-1] + [0] * 23, np.zeros((24, 3)), device="cpu")


def test_heading_draws_match_the_reference_protocol():
    from pulse_b200.motion_dataset import MotionDatasetB200
    z = load_npz("loader.npz")
    np.random.seed(4321)                       # whatever the caller's numpy state is, the worker re-seeds (pid 0 -> seed 0)
    h = MotionDatasetB200.draw_headings(len(z["headings"]))
    assert np.array_equal(h, z["headings"].numpy())


def test_selection_and_sampling_weights():
    ds = _dataset()
    ids = ds.select(10, random_sample=False, start_idx=4)
    assert ids.tolist() == [4, 5, 0, 1, 2, 3, 4, 5, 0, 1] and list(ds.curr_motion_keys[:3]) == ["clip_04", "clip_05", "clip_00"]
    ds.update_hard_sampling_weight(["clip_01", "clip_03"])
    assert torch.allclose(ds._sampling_prob, torch.tensor([0, 0.5, 0, 0.5, 0, 0]))
    torch.manual_seed(0)
    assert set(ds.select(50, random_sample=True).tolist()) == {1, 3}
    ds.update_hard_sampling_weight([])
    assert torch.allclose(ds._sampling_prob, torch.full((6,), 1 / 6))
    ds.update_soft_sampling_weight(["clip_02"])
    ds.update_soft_sampling_weight(["clip_02", "clip_05"])
    assert torch.allclose(ds._sampling_prob, torch.tensor([0, 0, 2 / 3, 0, 0, 1 / 3]))
    assert ds.update_sampling_prob(torch.zeros(6)) is False and ds.update_sampling_prob(torch.ones(5)) is False
    short = ds.crop(ds._motion_data_list[5], max_len=4)
    assert len(short["pose_quat_global"]) == 4 and len(short["root_trans_offset"]) == 4
    assert ds.crop(ds._motion_data_list[0], max_len=-1) is ds._motion_data_list[0]


def test_sampling_weights_against_reference_pins():
    """PMCP soft / hard sampling-weight updates against what the reference's MotionLibBase methods computed for the same
    sequence of failed clips (tests/golden/reference_pins.npz, make_golden_reference_pins.py)."""
    g = load_npz("reference_pins.npz")
    ds = _dataset()
    for i, failed in enumerate((["clip_02"], ["clip_02", "clip_05"], [], ["clip_00", "clip_01", "clip_04"])):
        ds.update_soft_sampling_weight(failed)
        assert torch.allclose(ds._sampling_prob, g[f"soft_prob_{i}"].float())
    for i, failed in enumerate((["clip_03"], [], ["clip_01", "clip_05"])):
        ds.update_hard_sampling_weight(failed)
        assert torch.allclose(ds._sampling_prob, g[f"hard_prob_{i}"].float())
