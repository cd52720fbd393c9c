"""pulse_b200 -- H100-native (sm_90a) implementation of PULSE's per-step rollout / update hot path.

Host code is Python/PyTorch (device memory, streams, torch.distributed) calling hand-written CUDA
through the C ABI in include/pulse_b200.h (libpulse_b200.so, built in-tree by pulse_b200.build).
There is no CPU fallback: importing the compute modules without the built library fails loudly.
"""
from . import _lib  # noqa: F401
from ._lib import PulseError  # noqa: F401

__all__ = ["ImZStepsB200", "PulseError", "TerrainResetB200", "TerrainStepsB200", "ZTaskStepsB200"]


def __getattr__(name):
    if name == "ZTaskStepsB200":           # resolved on first use: importing the package alone does not import torch
        from .ztask_rollout import ZTaskStepsB200
        return ZTaskStepsB200
    if name == "TerrainStepsB200":
        from .terrain_rollout import TerrainStepsB200
        return TerrainStepsB200
    if name == "ImZStepsB200":
        from .imz_rollout import ImZStepsB200
        return ImZStepsB200
    if name == "TerrainResetB200":
        from .terrain_reset import TerrainResetB200
        return TerrainResetB200
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
__version__ = "0.1.0"
