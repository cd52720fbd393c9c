"""Import the UNMODIFIED reference tree (PULSE_REFERENCE_ROOT) for fixture generation.

TEST INFRASTRUCTURE ONLY.  The reference's hot-path functions are plain PyTorch, but the modules
that hold them import Isaac Gym, rl_games, smpl_sim, ... at module scope.  This loader registers
(a) the file-based `isaacgym.torch_utils` restatement next to this file and (b) attribute-mocks
for every other missing third-party module, then imports the reference modules as they are.

Used only by the fixture generators under `tests/golden/` (`make_golden*.py`): the tests compare against the
fixtures they wrote and never import the reference.  The reference tree's location is PULSE_REFERENCE_ROOT.
"""
import importlib
import importlib.abc
import importlib.machinery
import os
import sys
import types
from unittest.mock import MagicMock

REFERENCE_ROOT = os.environ.get("PULSE_REFERENCE_ROOT", "/root/reference")
_SHIM_DIR = os.path.dirname(os.path.abspath(__file__))


class _Mock(types.ModuleType):
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        m = MagicMock(name=f"{self.__name__}.{name}")
        setattr(self, name, m)
        return m


class _EasyDict(dict):
    """Attribute dictionary (enough of `easydict.EasyDict` for MotionLibBase.__init__)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


# Top-level third-party packages the reference imports at module scope and that are absent here.
# Any submodule of these resolves to an attribute-mock through the meta-path finder below.
_MOCK_TOPS = [
    "smpl_sim", "easydict", "open3d", "imageio", "rl_games", "gym", "aiohttp", "termcolor",
    "pyvirtualdisplay", "skimage", "mujoco", "lxml", "wandb", "tensorboardX", "horovod", "sru",
    "cv2", "ipdb", "hydra", "omegaconf", "vtk", "chumpy", "smplx", "matplotlib", "mpl_toolkits",
    "gymnasium", "trimesh", "pyrender",
]
_ISAAC_SUBS = ("gymapi", "gymtorch", "gymutil", "terrain_utils")


class _MockFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def __init__(self, tops):
        self.tops = set(tops)

    def find_spec(self, fullname, path, target=None):
        top = fullname.split(".")[0]
        if top in self.tops or (top == "isaacgym" and fullname.split(".")[-1] in _ISAAC_SUBS):
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        return _Mock(spec.name)

    def exec_module(self, module):
        pass


def _missing(name):
    try:
        importlib.import_module(name)
        return False
    except Exception:
        return True


_loaded = {}


def load_reference():
    """Returns a namespace with the reference modules on the hot path."""
    if _loaded:
        return types.SimpleNamespace(**_loaded)
    if not os.path.isdir(REFERENCE_ROOT):
        raise FileNotFoundError(f"reference tree not found at {REFERENCE_ROOT}")
    for p in (REFERENCE_ROOT, os.path.join(REFERENCE_ROOT, "phc"), _SHIM_DIR):
        if p in sys.path:
            sys.path.remove(p)
    # `phc/` itself goes on the path because the reference imports `learning.*` as a top-level
    # package (it is launched from inside the tree with cwd on sys.path).
    sys.path[:0] = [_SHIM_DIR, REFERENCE_ROOT, os.path.join(REFERENCE_ROOT, "phc")]

    import isaacgym  # the shim package next to this file
    tops = [t for t in _MOCK_TOPS if _missing(t)]
    sys.meta_path.append(_MockFinder(tops))
    for sub in _ISAAC_SUBS:
        setattr(isaacgym, sub, importlib.import_module(f"isaacgym.{sub}"))
    importlib.import_module("easydict").EasyDict = _EasyDict

    import numpy as np
    import torch

    def _to_torch(x):
        return x if torch.is_tensor(x) else torch.from_numpy(np.asarray(x))

    importlib.import_module("smpl_sim.utils.torch_ext").to_torch = _to_torch

    mods = {}
    mods["flags"] = importlib.import_module("phc.utils.flags").flags
    for attr, val in (("test", False), ("im_eval", False), ("debug", False), ("real_traj", False),
                      ("server_mode", False), ("render_o3d", False), ("no_collision_check", False)):
        setattr(mods["flags"], attr, val)
    mods["torch_utils"] = importlib.import_module("phc.utils.torch_utils")
    mods["motion_lib_base"] = importlib.import_module("phc.utils.motion_lib_base")
    mods["motion_lib_smpl"] = importlib.import_module("phc.utils.motion_lib_smpl")
    mods["humanoid"] = importlib.import_module("phc.env.tasks.humanoid")
    mods["humanoid_amp"] = importlib.import_module("phc.env.tasks.humanoid_amp")
    mods["humanoid_im"] = importlib.import_module("phc.env.tasks.humanoid_im")
    mods["running_mean_std"] = importlib.import_module("phc.utils.running_mean_std")
    mods["loss_functions"] = importlib.import_module("phc.learning.loss_functions")
    mods["skeleton3d"] = importlib.import_module("poselib.poselib.skeleton.skeleton3d")
    mods["EasyDict"] = _EasyDict
    _loaded.update(mods)
    return types.SimpleNamespace(**mods)


_learning = {}


def load_learning():
    """Import the reference's agent / network modules (phc/learning).

    rl_games 1.1.4 is absent, so the base classes the reference subclasses are replaced by empty
    real classes (a MagicMock cannot be subclassed into a usable class).  Only methods defined in
    the reference's own files are exercised: `discount_values`, `_actor_loss`, `_critic_loss`,
    `bound_loss`, `_calc_advs` (common_agent.py), `_disc_loss*`, `_calc_disc_rewards`
    (amp_agent.py) and the in-tree network builders.
    """
    if _learning:
        return types.SimpleNamespace(**_learning)
    load_reference()
    import torch.nn as nn

    class _Anything:
        def __init__(self, *a, **k):
            pass

    def _stub(modname, clsname, base=_Anything, **attrs):
        mod = importlib.import_module(modname)
        cls = type(clsname, (base,), dict(attrs))
        setattr(mod, clsname, cls)
        return cls

    _stub("rl_games.algos_torch.a2c_continuous", "A2CAgent")
    _stub("rl_games.algos_torch.a2c_discrete", "DiscreteA2CAgent")
    _stub("rl_games.common.datasets", "PPODataset")
    _stub("rl_games.common.player", "BasePlayer")
    _stub("rl_games.algos_torch.players", "PpoPlayerContinuous")
    base_model = _stub("rl_games.algos_torch.models", "ModelA2CContinuousLogStd")
    base_model.Network = type("Network", (nn.Module,), {})

    mods = {}
    for key, name in (("common_agent", "learning.common_agent"), ("amp_agent", "learning.amp_agent"),
                      ("network_builder", "phc.learning.network_builder"),
                      ("amp_network_builder", "learning.amp_network_builder"),
                      ("amp_network_z_builder", "phc.learning.amp_network_z_builder"),
                      ("amp_datasets", "learning.amp_datasets"),
                      ("replay_buffer", "learning.replay_buffer")):
        mods[key] = importlib.import_module(name)
    _learning.update(mods)
    return types.SimpleNamespace(**mods)


if __name__ == "__main__":
    ref = load_reference()
    print("reference imported:", sorted(vars(ref)))
    lrn = load_learning()
    print("learning imported:", sorted(vars(lrn)))
