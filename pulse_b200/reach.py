"""Downstream latent-space reach task (SURVEY K21, BASELINE config 5): host-side mirror of
`phc.env.tasks.humanoid_reach.HumanoidReach` / `HumanoidReachZ` (humanoid_reach.py:17-166, :224-250) for the
post-physics path -- reward, reset, observation -- and the target resampling of `_update_task` / `_reset_task`.

The step object lives in `pulse_b200.ztasks` with the speed and strike tasks' and shares their base; this module keeps its names.
"""
from .ztasks import REACH_OBS, SMPL_BODY_NAMES, ReachTaskB200

__all__ = ["REACH_OBS", "SMPL_BODY_NAMES", "ReachTaskB200"]
