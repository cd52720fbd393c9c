"""Pedestrian terrain task: the oracle's restatement (oracle/terrain_oracle.py) against the fixture written by the UNMODIFIED reference
(tests/golden/make_golden_terrain.py) -- integers identical, floats within 2e-6 -- and the C ABI of the new entry points."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import terrain_oracle as to

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DT = 2 * (1.0 / 60.0)
MAX_LEN = 300
CONTACT_IDS = [7, 3, 8, 4]


def gen():
    spec = importlib.util.spec_from_file_location("make_golden_terrain", os.path.join(HERE, "golden", "make_golden_terrain.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


CASES = gen().CASES


def fixture(case="a"):
    """The reference's outputs with the inputs of `case` (its first n envs) rebuilt from their seeds."""
    m = gen()
    g = np.load(os.path.join(HERE, "golden", "terrain.npz"))
    z = {k: torch.from_numpy(g[k]) for k in g.files}
    z.update(m.case_inputs(m.inputs(), CASES[case]["n"]))
    return z


def cell_heights(z) -> torch.Tensor:
    """The reference's head-pose heights from its cells: min(hf[px, py], hf[px + 1, py + 1]) * vertical_scale (:1262-1267)."""
    px, py, hf = z["a_px"].long(), z["a_py"].long(), z["heightfield"]
    return torch.min(hf[px, py], hf[px + 1, py + 1]) * 0.005


def close(a, b, name, tol=2e-6):
    torch.testing.assert_close(a, b, atol=tol, rtol=tol, msg=lambda s: f"{name}: {s}")


def test_trajectory_matches_reference():
    m, g = gen(), fixture()
    draws, init = m.reset_draws()
    n = draws.shape[0]
    traj_dt = to.traj_params(MAX_LEN, DT)
    verts = torch.zeros(n, to.TRAJ_VERTS, 3)
    to.traj_reset(verts, torch.arange(n), init, draws, traj_dt, 2.0, 0.0, 3.0, 2.0, 0.02)
    close(verts, g["traj_reset_verts"], "traj_verts")
    t = m.CALC_POS_TIMES
    pos = to.traj_calc_pos(g["traj_reset_verts"], torch.arange(n).repeat_interleave(len(t)), t.repeat(n), traj_dt).view(n, len(t), 3)
    close(pos, g["calc_pos"], "calc_pos")


def test_height_cells_match_reference():
    g = fixture()
    head = g["body_state"][:, to.HEAD_BODY_ID, 0:7]
    pts = to.grid_points_world(head, to.square_height_points(), True)
    px, py = to.world_points_to_map(pts, 0.1, *g["heightfield"].shape)
    assert torch.equal(px.view_as(g["a_px"]), g["a_px"].long()) and torch.equal(py.view_as(g["a_py"]), g["a_py"].long())
    assert int(px.min()) == 0 and int(px.max()) == g["heightfield"].shape[0] - 2     # the fixture exercises both clips
    close(to.grid_heights(g["heightfield"], 0.1, 0.005, head, to.square_height_points(), True), cell_heights(g), "heights")


@pytest.mark.parametrize("case", sorted(CASES))
def test_step_matches_reference(case):
    g = fixture(case)
    c = CASES[case]
    hf = g["heightfield"]
    bs = g["body_state"]
    out = to.terrain_step(hf, 0.1, 0.005, bs, g["root_states"], g["progress_buf"], g["contact_forces"], torch.tensor(CONTACT_IDS),
                          g["dof_force"], g["dof_vel"], g["traj_verts"], dt=DT, traj_dt=to.traj_params(MAX_LEN, DT), max_episode_length=MAX_LEN,
                          upright=c["upright"], fuzzy=c["fuzzy"], power_reward=c["power"], use_center_height=c["use_center_height"])
    assert torch.equal(out["reset"], g[f"{case}_reset"]) and torch.equal(out["terminate"], g[f"{case}_terminate"])
    assert 0 < int(out["terminate"].sum()) < len(out["terminate"])
    close(out["rew"], g[f"{case}_rew"], "rew")
    close(out["reward_raw"], g[f"{case}_reward_raw"], "reward_raw", 2e-5)   # |power| ~ 1: fp32 sums over 69 dofs in another order
    close(out["obs"][:, :358], g[f"{case}_self_obs"], "self_obs")
    close(out["obs"][:, 358:], g[f"{case}_task_obs"], "task_obs")
    close(to.center_heights(hf, 0.1, 0.005, bs[:, 0, 0:7], to.center_height_points(), c["upright"]), g[f"{case}_center_heights"], "center")
    close(to.center_heights(hf, 0.1, 0.005, g["root_states"][:, 0:7], to.center_height_points(), c["upright"]), g[f"{case}_root_center_heights"],
          "root center")


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def test_terrain_struct_sizes_match_header(lib):
    import subprocess
    import tempfile
    from pulse_b200 import _lib
    src = ('#include <stdio.h>\n#include "pulse_b200.h"\nint main(){printf("%zu %zu %zu %d %d %d\\n", sizeof(pulse_terrain_step_args_t), '
           'sizeof(pulse_traj_reset_args_t), sizeof(pulse_terrain_heights_args_t), PULSE_TRAJ_VERTS, PULSE_TRAJ_DRAWS, PULSE_TERRAIN_OBS);return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    from pulse_b200.terrain import TERRAIN_OBS
    assert got == [C.sizeof(_lib.TerrainStepArgs), C.sizeof(_lib.TrajResetArgs), C.sizeof(_lib.TerrainHeightsArgs), _lib.TRAJ_VERTS,
                   _lib.TRAJ_DRAWS, TERRAIN_OBS]


def test_terrain_entry_points_validate_arguments_without_gpu(lib):
    from pulse_b200 import _lib
    assert lib.pulse_terrain_step(None, 4, None) == -1 and b"null" in lib.pulse_last_error()
    buf = (C.c_float * 64)()
    ptr = C.cast(buf, C.c_void_p)
    a = _lib.TerrainStepArgs(flags=16)
    assert lib.pulse_terrain_step(C.byref(a), 4, None) == -1 and b"flags" in lib.pulse_last_error()
    a = _lib.TerrainStepArgs(flags=_lib.STEP_ALL, body_state=ptr, body_env_stride=312, root_states=ptr, root_env_stride=13, progress_buf=ptr,
                             traj_verts=ptr, dt=1 / 30, traj_dur=10.1, rew_buf=ptr, reward_raw=ptr, raw_stride=2)
    assert lib.pulse_terrain_step(C.byref(a), 4, None) == -1 and b"dof_force" in lib.pulse_last_error()
    a.reward_raw = None
    assert lib.pulse_terrain_step(C.byref(a), 4, None) == -1 and b"reset_buf" in lib.pulse_last_error()
    a.reset_buf = a.terminate_buf = ptr
    a.enable_early_termination = 1
    assert lib.pulse_terrain_step(C.byref(a), 4, None) == -1 and b"contact_forces" in lib.pulse_last_error()
    a.enable_early_termination = 0
    a.obs_buf, a.height_points, a.center_points, a.num_traj_samples, a.num_height_points, a.num_center_points = ptr, ptr, ptr, 10, 1024, 9
    a.head_body_id, a.obs_stride = 13, 1000
    assert lib.pulse_terrain_step(C.byref(a), 4, None) == -1 and b"obs_stride" in lib.pulse_last_error()
    a.obs_stride, a.heightfield, a.hf_rows, a.hf_cols = 1402, ptr, 1, 5
    assert lib.pulse_terrain_step(C.byref(a), 4, None) == -1 and b"2 x 2" in lib.pulse_last_error()
    a.env_ids = ptr
    assert lib.pulse_terrain_step(C.byref(a), 4, None) == -1 and b"env_ids" in lib.pulse_last_error()
    t = _lib.TrajResetArgs(num_ids=3)
    assert lib.pulse_traj_reset(C.byref(t), None) == -1 and b"null" in lib.pulse_last_error()
    t.num_ids = 0
    assert lib.pulse_traj_reset(C.byref(t), None) == 0                    # nothing to reset: no launch
    h = _lib.TerrainHeightsArgs(mode=3)
    assert lib.pulse_terrain_heights(C.byref(h), None) == -1 and b"mode" in lib.pulse_last_error()


def test_mixin_refuses_unsupported_options_without_gpu():
    from pulse_b200.terrain import check_terrain_options, PulseError
    ok = dict(cfg={"env": {"terrain": {"terrainType": "trimesh"}}}, _divide_group=False, _group_obs=False, velocity_map=False, real_mesh=False,
              _has_shape_obs=False, big_ankle=False)
    check_terrain_options(_ns(**ok), _ns(server_mode=False, real_path=False, fixed_path=False, slow=False))
    for key, val, word in (("_divide_group", True, "divide_group"), ("_group_obs", True, "group_obs"), ("velocity_map", True, "velocity_map"),
                           ("real_mesh", True, "real_mesh"), ("_has_shape_obs", True, "has_shape_obs"), ("big_ankle", True, "big_ankle")):
        with pytest.raises(PulseError, match=word):
            check_terrain_options(_ns(**{**ok, key: val}), _ns(server_mode=False, real_path=False, fixed_path=False, slow=False))
    for flag in ("server_mode", "real_path", "fixed_path", "slow"):
        f = dict(server_mode=False, real_path=False, fixed_path=False, slow=False)
        f[flag] = True
        with pytest.raises(PulseError, match=flag):
            check_terrain_options(_ns(**ok), _ns(**f))


def _ns(**kw):
    import types
    return types.SimpleNamespace(**kw)
