"""Host side of the evaluation pass (`EvalStepsB200`, pulse_b200/evaluation.py) without a GPU: the chunk schedule against the reference's
formulas (clip ids by `torch.remainder`, motion_lib_base.py:208; `bound`, im_amp.py:254-256; the pass ends at the chunk with
start_idx + N >= U, im_amp.py:295), the chunk loop driven through the block callback against the per-step one, the step configuration
of a pass (`eval_config`) and the task settings of im_amp.py:160-182 applied and put back by `eval_settings` on a stand-in task."""
import dataclasses
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from pulse_b200 import _lib
from pulse_b200.evaluation import (ALL_BODIES, EvalLoopB200, chunk_bound, chunk_clip_ids, chunk_starts, eval_config, eval_settings)
from tests.test_eval_host_cpu import NumpyMetrics, Sim

CASES = [(64, 150), (64, 64), (64, 65), (16384, 11313), (7, 3), (1, 1), (5, 21), (100, 99)]


def _reference_schedule(N, U):
    """begin_seq_motion_samples / forward_motion_samples / the end test of _post_step_eval, as the reference runs them."""
    out, start_idx = [], 0
    while True:
        curr_ids = torch.remainder(torch.arange(N) + start_idx, U)                         # motion_lib_base.py:208
        max_possible_id = U - 1
        bound = int((max_possible_id == curr_ids).nonzero()[0]) + 1 if (max_possible_id == curr_ids).sum() > 0 else N
        out.append((start_idx, curr_ids.numpy(), bound))
        if start_idx + N >= U:                                                              # im_amp.py:295
            return out
        start_idx += N                                                                      # humanoid_im.py:445-447


@pytest.mark.parametrize("N,U", CASES)
def test_chunk_schedule_matches_reference(N, U):
    ref = _reference_schedule(N, U)
    starts = chunk_starts(N, U)
    assert starts == [s for s, _, _ in ref]
    assert len(starts) == -(-U // N)
    for s, ids, bound in ref:
        got = chunk_clip_ids(s, N, U)
        assert np.array_equal(got, ids)
        assert chunk_bound(got, U) == bound
    covered = np.concatenate([chunk_clip_ids(s, N, U) for s in starts])[:U]                  # the first U sequences are every clip once
    assert np.array_equal(covered, np.arange(U))


@pytest.mark.parametrize("N,U", [(8, 21), (8, 5)])
def test_dataset_select_is_the_chunk_schedule(N, U):
    from pulse_b200.motion_dataset import MotionDatasetB200
    clips = {f"clip_{i:02d}": {"pose_quat_global": np.zeros((4, 24, 4))} for i in range(U)}
    ds = MotionDatasetB200(clips, list(range(-1, 23)), np.zeros((24, 3)), device="cpu")
    for s in chunk_starts(N, U):
        ds.select(N, random_sample=False, start_idx=s)
        assert np.array_equal(ds._curr_motion_ids.numpy(), chunk_clip_ids(s, N, U))


@pytest.mark.parametrize("N,U,poll", [(16, 40, 1), (16, 40, 5), (8, 16, 8), (32, 20, 3), (4, 9, 2)])
def test_block_callback_matches_per_step_loop(N, U, poll):
    """`steps` runs `poll_every` steps per call (steps past a chunk's end are no-ops in the metrics) and ends every chunk where the
    per-step loop does."""
    sim = Sim(N, U, seed=N * 7 + U)
    a = EvalLoopB200(N, U, sim.keys, load_chunk=sim.load_chunk, reset_all=lambda: None, step=sim.frame, poll_every=poll,
                     metrics=NumpyMetrics(N)).run()
    sim2, m = Sim(N, U, seed=N * 7 + U), NumpyMetrics(N)
    calls = []

    def steps():
        calls.append(1)
        for _ in range(poll):
            m.step(*sim2.frame())

    b = EvalLoopB200(N, U, sim2.keys, load_chunk=sim2.load_chunk, reset_all=lambda: None, steps=steps, poll_every=poll, metrics=m).run()
    assert a["steps"] == b["steps"] and a["chunks"] == b["chunks"] == len(chunk_starts(N, U))
    assert np.array_equal(a["terminated"], b["terminated"])
    assert a["eval_info"] == b["eval_info"]
    assert len(calls) * poll >= b["steps"]


def test_loop_takes_one_step_callback():
    for kw in ({}, {"step": lambda: None, "steps": lambda: None}):
        with pytest.raises(_lib.PulseError, match="one of step / steps"):
            EvalLoopB200(4, 9, [str(i) for i in range(9)], load_chunk=None, reset_all=None, metrics=NumpyMetrics(4), **kw)


def test_eval_config():
    from pulse_b200.humanoid_im import DEFAULT_RESET_BODIES, ImConfig
    im = ImConfig(cycle_motion=True)
    vr = ImConfig(reset_body_ids=(13, 18, 23), track_body_ids=(13, 18, 23), termination_distance=0.25)
    before = (dataclasses.asdict(im), dataclasses.asdict(vr))
    e = eval_config(im)
    assert len(DEFAULT_RESET_BODIES) == 20 and tuple(e.reset_body_ids) == ALL_BODIES == tuple(range(24))    # > 15 reset bodies: swapped
    assert e.termination_distance == 0.5 and e.use_mean_reset and not e.cycle_motion
    v = eval_config(vr)
    assert tuple(v.reset_body_ids) == (13, 18, 23) and tuple(v.track_body_ids) == (13, 18, 23)               # three-point tracking: kept
    assert v.termination_distance == 0.5 and v.use_mean_reset
    assert not eval_config(im, strict_eval=True).use_mean_reset                                              # im_eval and not strict_eval
    assert tuple(eval_config(im, eval_body_ids=(0, 5, 9)).reset_body_ids) == (0, 5, 9)
    assert (dataclasses.asdict(im), dataclasses.asdict(vr)) == before                                        # the training configs are not touched


def _task(n_reset, getup):
    t = NS(_termination_distances=torch.full((1, 24), 0.25), cycle_motion=True, zero_out_far=True,
           _reset_bodies_id=torch.arange(n_reset), _eval_track_bodies_id=torch.arange(24) + 100, _pulse_im_eval=False)
    if getup:
        t._recovery_episode_prob, t._fall_init_prob = 0.2, 0.1
    return t


@pytest.mark.parametrize("n_reset,getup", [(20, False), (3, False), (24, True)])
def test_eval_settings_applied_and_restored(n_reset, getup):
    flags = NS(test=False, im_eval=False)
    task = _task(n_reset, getup)
    reset_ids = task._reset_bodies_id
    dist = task._termination_distances
    with eval_settings(task, flags=flags) as t:
        assert t is task and flags.test and flags.im_eval and task._pulse_im_eval
        assert task._termination_distances is dist and bool((dist == 0.5).all())                            # in place, like [:] = 0.5
        assert not task.cycle_motion and not task.zero_out_far
        if n_reset > 15:
            assert task._reset_bodies_id is task._eval_track_bodies_id
        else:
            assert task._reset_bodies_id is reset_ids
        if getup:
            assert task._recovery_episode_prob == 0 and task._fall_init_prob == 0
    assert task._termination_distances is dist and bool((dist == 0.25).all())
    assert task.cycle_motion and task.zero_out_far and task._reset_bodies_id is reset_ids and not task._pulse_im_eval
    assert not flags.test and not flags.im_eval
    if getup:
        assert task._recovery_episode_prob == 0.2 and task._fall_init_prob == 0.1
    else:
        assert "_recovery_episode_prob" not in task.__dict__


def test_eval_settings_restored_on_error():
    flags = NS(test=False, im_eval=False)
    task = _task(20, True)
    with pytest.raises(RuntimeError):
        with eval_settings(task, flags=flags):
            raise RuntimeError("pass failed")
    assert bool((task._termination_distances == 0.25).all()) and task.cycle_motion and task._recovery_episode_prob == 0.2
    assert len(task._reset_bodies_id) == 20 and not flags.test and not flags.im_eval


def test_eval_steps_refuses_other_drivers():
    from pulse_b200.evaluation import EvalStepsB200
    with pytest.raises(_lib.PulseError, match="PlayStepsB200 and ImZStepsB200"):
        EvalStepsB200(NS(policy=None))
