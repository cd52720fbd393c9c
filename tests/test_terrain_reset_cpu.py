"""CPU checks of the pedestrian terrain task's reset: the oracle (tests/terrain_reset_oracle.py) against the unmodified reference's
`_reset_ref_state_init` / `sample_valid_locations` / `get_center_heights` / `_init_amp_obs` recorded in tests/golden/terrain_reset.npz,
the C ABI and argument checks of `pulse_reset_terrain` / `pulse_traj_reset_list`, the Philox keying of the list trajectory reset, and
the mixin's refusals."""
import ctypes as C
import os
import types

import pytest
import torch

from oracle import pulse_oracle as po
from oracle import terrain_oracle as to
from tests import terrain_reset_oracle as tro
from tests import ztask_reset_oracle as zo
from tests.helpers import load_npz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"upright": True, "tilted": False, "start": True}
N = 48


@pytest.fixture(scope="module")
def fx():
    return load_npz("terrain_reset.npz")


@pytest.fixture(scope="module")
def tables():
    from pulse_b200.ztask_reset import smpl_ground_table
    tb, betas = zo.fixture_tables()
    return tb, smpl_ground_table(tb.motion_aa, zo.StandInParser(), betas)


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


def heightfield():
    from tests.golden.make_golden_terrain import heightfield as hf
    return torch.from_numpy(hf())


def injected(fx, case):
    ids = fx[case + "_env_ids"]
    assert str(fx[case + "_draws"]).split() == ["multinomial", "rand", "randint"]     # _sample_time for StateInit Start too
    d = {"motion_ids": torch.zeros(N, dtype=torch.int64), "phase": torch.zeros(N), "loc_ids": torch.zeros(N, dtype=torch.int64)}
    d["motion_ids"][ids], d["phase"][ids], d["loc_ids"][ids] = fx[case + "_draw0"], fx[case + "_draw1"], fx[case + "_draw2"].long()
    return ids, d


def zero_state():
    return {"root_states": torch.zeros(N, 13), "dof_pos": torch.zeros(N, 69), "dof_vel": torch.zeros(N, 69), "body_state": torch.zeros(N, 24, 13),
            "sampled_motion_ids": torch.zeros(N, dtype=torch.int64), "motion_start_times": torch.zeros(N),
            "progress_buf": torch.zeros(N, dtype=torch.int64), "reset_buf": torch.zeros(N, dtype=torch.int64),
            "terminate_buf": torch.zeros(N, dtype=torch.int64), "contact_forces": torch.zeros(N, 24, 3), "amp_obs_buf": torch.zeros(N, 10, 196)}


def test_walkable_table_restatement_is_the_fixtures(fx):
    from tests.golden.make_golden_terrain_reset import BORDER
    cx, cy = tro.walkable_table(tro.walkable_field(*heightfield().shape), 0.1, BORDER)
    assert torch.equal(cx, fx["coord_x"]) and torch.equal(cy, fx["coord_y"])


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reproduces_reference_reset(fx, tables, case):
    """Clips, start times and location indices exactly; states, AMP rows and the spawn's center points within 2e-6 of the reference,
    which lifts each pose with the parser's mesh instead of the floor table."""
    tb, floor = tables
    ids, d = injected(fx, case)
    hf = heightfield()
    o = tro.terrain_reset(tb, zero_state(), ids, d, floor, hf, fx["coord_x"], fx["coord_y"], upright=CASES[case])
    assert torch.equal(o["sampled_motion_ids"][ids], fx[case + "_ref_motion_ids"])
    assert torch.equal(o["motion_start_times"][ids], fx[case + "_ref_motion_times"])
    # the reference's terrain reset does not write _sampled_motion_ids / _motion_start_times: the mixin hands the kernel its own
    assert not fx[case + "_motion_ids"].any() and not fx[case + "_start_times"].any()
    for k, ref in (("root_states", "root_states"), ("dof_pos", "dof_pos"), ("dof_vel", "dof_vel"), ("body_state", "body_state"),
                   ("amp_obs_buf", "amp_obs")):
        torch.testing.assert_close(o[k], fx[case + "_" + ref], rtol=0, atol=2e-6, msg=lambda m: f"{case} {k}: {m}")
    rs = o["root_states"][ids]
    pts = to.center_points_world(torch.cat([rs[:, 0:3], rs[:, 3:7]], dim=-1), to.center_height_points(), CASES[case])
    torch.testing.assert_close(pts[..., 0:2], fx[case + "_center_points_world"][..., 0:2], rtol=0, atol=2e-6)


def test_fixture_covers_the_edge_cases(fx):
    """Upright and tilted roots, a yaw within 0.2 of pi, spawn points on cell boundaries (every walkable coordinate is a cell corner),
    center points on slopes and steps (the nine heights of one spawn differ), and reset sets holding env 0 and env N - 1."""
    hf = heightfield()
    assert not torch.allclose(fx["tilted_root_states"], fx["upright_root_states"])
    big_yaw = 0.0
    for case, upright in CASES.items():
        ids = fx[case + "_env_ids"]
        assert int(ids[0]) == 0 and int(ids[-1]) == N - 1
        rs = fx[case + "_root_states"][ids]
        h = po.heading_quat(rs[:, 3:7] if upright else po.remove_base_rot(rs[:, 3:7]))
        big_yaw = max(big_yaw, float((2 * torch.atan2(h[:, 2], h[:, 3])).remainder(2 * torch.pi).sub(torch.pi).abs().min().neg().add(torch.pi)))
        w = fx[case + "_center_points_world"]
        cells = w[:, 4, 0:2] / 0.1                                          # the middle point is the spawn point itself
        assert float((cells - cells.round()).abs().max()) < 1e-3
        heights = to.sample_height_points(hf, w, 0.1, 0.005)
        assert int((heights.max(dim=-1).values > heights.min(dim=-1).values).sum()) >= 3
    assert big_yaw > torch.pi - 0.2


def test_reset_task_restates_the_trajectory_generator():
    """The list trajectory reset of the oracle is TrajGenerator.reset at the new roots (the generator itself is pinned by terrain.npz)."""
    g = torch.Generator().manual_seed(3)
    roots = torch.randn(6, 13, generator=g)
    rand = torch.rand(6, to.TRAJ_DRAWS, generator=g)
    v = tro.reset_task(torch.zeros(6, to.TRAJ_VERTS, 3), torch.tensor([1, 4]), roots, rand)
    assert torch.equal(v[[0, 2, 3, 5]], torch.zeros(4, to.TRAJ_VERTS, 3))
    assert torch.equal(v[[1, 4], 0, 0:2], roots[[1, 4], 0:2])


def test_terrain_reset_symbols_and_struct_layout(lib):
    import subprocess
    import tempfile
    from pulse_b200 import _lib
    for n in ("pulse_reset_terrain", "pulse_traj_reset_list"):
        assert hasattr(lib, n) and n in _lib.SIGNATURES
    assert lib.pulse_abi_version() == 3
    sf = ("hf_rows", "horizontal_scale", "center_points", "num_center_points", "coord_x", "coord_y", "num_locations", "loc_ids_in", "loc_ids_out")
    lf = ("count", "root_states", "root_env_stride", "rand", "seed", "offset_dev", "dtheta_scale", "sharp_turn_prob", "verts")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "pulse_b200.h"\nint main(){printf("%zu %zu %zu %zu", '
           'sizeof(pulse_terrain_spawn_args_t), sizeof(pulse_traj_list_args_t), sizeof(pulse_ztask_reset_args_t), sizeof(pulse_traj_reset_args_t));'
           + "".join(f'printf(" %zu", offsetof(pulse_terrain_spawn_args_t, {f}));' for f in sf)
           + "".join(f'printf(" %zu", offsetof(pulse_traj_list_args_t, {f}));' for f in lf) + "return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert got == ([C.sizeof(_lib.TerrainSpawnArgs), C.sizeof(_lib.TrajListArgs), C.sizeof(_lib.ZTaskResetArgs), C.sizeof(_lib.TrajResetArgs)]
                   + [getattr(_lib.TerrainSpawnArgs, f).offset for f in sf] + [getattr(_lib.TrajListArgs, f).offset for f in lf])


def _valid(_lib, ptr):
    a = _lib.ZTaskResetArgs()
    a.reset_buf = a.env_list = a.count = ptr
    a.sampled_motion_ids = a.motion_start_times = a.progress_buf = ptr
    a.root_states = a.dof_pos = a.dof_vel = a.rigid_body_state = ptr
    a.root_env_stride, a.dof_env_stride, a.dof_elem_stride, a.body_env_stride = 13, 138, 2, 312
    a.floor, a.floor_len, a.sampling_cdf = ptr, 10, ptr
    s = _lib.TerrainSpawnArgs(heightfield=ptr, hf_rows=4, hf_cols=4, horizontal_scale=0.1, vertical_scale=0.005, center_points=ptr,
                              num_center_points=9, coord_x=ptr, coord_y=ptr, num_locations=5)
    return a, s


def test_terrain_entry_points_validate_arguments_without_gpu(lib):
    """Every refusal happens before anything touches the device, so a CPU-only machine exercises them all."""
    from pulse_b200 import _lib
    buf = (C.c_float * 256)()
    ptr = C.cast(buf, C.c_void_p)
    desc = _lib.MotionLibDesc(aux_rec=ptr, total_frames=10, num_motions=2)
    fake_lib = C.cast(C.pointer(desc), C.c_void_p)
    a, s = _valid(_lib, ptr)
    assert lib.pulse_reset_terrain(fake_lib, C.byref(a), None, 4, None) == -1 and b"null" in lib.pulse_last_error()

    def refuses(change, words):
        a, s = _valid(_lib, ptr)
        change(a, s)
        assert lib.pulse_reset_terrain(fake_lib, C.byref(a), C.byref(s), 4, None) == -1
        assert words.encode() in lib.pulse_last_error(), lib.pulse_last_error()

    refuses(lambda a, s: setattr(a, "reset_buf", None), "mask")
    refuses(lambda a, s: setattr(a, "count", None), "count outputs")
    refuses(lambda a, s: setattr(a, "rigid_body_state", None), "null simulator tensor")
    refuses(lambda a, s: setattr(a, "body_env_stride", 300), "strides")
    refuses(lambda a, s: (setattr(a, "target_states", ptr), setattr(a, "target_env_stride", 13)), "no target actor")
    refuses(lambda a, s: setattr(a, "floor_len", 9), "floor table of 9 frames")
    refuses(lambda a, s: setattr(a, "pose_mode", _lib.ZPOSE_FACE_X), "pose_mode")
    refuses(lambda a, s: setattr(a, "state_init", _lib.ZINIT_START), "always samples the start time")
    refuses(lambda a, s: (setattr(a, "amp_obs_buf", ptr), setattr(a, "num_amp_steps", 10), setattr(a, "amp_width", 194)), "amp_width 194")
    refuses(lambda a, s: setattr(s, "heightfield", None), "plane terrain")
    refuses(lambda a, s: setattr(s, "hf_rows", 1), "2 x 2 cells")
    refuses(lambda a, s: setattr(s, "num_center_points", 33), "num_center_points 33")
    refuses(lambda a, s: setattr(s, "num_locations", 0), "walkable table of 0 locations")
    refuses(lambda a, s: setattr(s, "coord_y", None), "walkable table")
    a, s = _valid(_lib, ptr)
    assert lib.pulse_reset_terrain(fake_lib, C.byref(a), C.byref(s), 0, None) == 0          # nothing to do: no launch

    t = _lib.TrajListArgs()
    assert lib.pulse_traj_reset_list(None, 4, None) == -1 and b"null args" in lib.pulse_last_error()
    assert lib.pulse_traj_reset_list(C.byref(t), 4, None) == -1 and b"null list" in lib.pulse_last_error()
    t.env_list = t.count = t.root_states = t.verts = ptr
    assert lib.pulse_traj_reset_list(C.byref(t), 4, None) == -1 and b"root_env_stride" in lib.pulse_last_error()
    t.root_env_stride = 13
    assert lib.pulse_traj_reset_list(C.byref(t), 4, None) == -1 and b"trajectory parameters" in lib.pulse_last_error()
    t.seg_dt, t.speed_max = 0.1, 3.0
    assert lib.pulse_traj_reset_list(C.byref(t), 0, None) == 0


@pytest.mark.parametrize("first,second", [((0, 0), (1, 0)), ((0, 0), (0, 1)), ((5, 3), (7, 2)), ((2 ** 40, 1), (2 ** 40 + 1, 1)),
                                          ((1, 0), (0, 0)), ((10, 0), (3, 6))])
def test_traj_list_philox_blocks_of_two_resets_are_disjoint(first, second):
    """Two trajectory resets of one env at different (offset + *offset_dev) read no common Philox block, also when a driver advances
    the device offset by one per step; and the list plane is apart from every index plane of the latent tasks."""
    from pulse_b200 import _lib
    i1, c1 = _lib.traj_list_philox_blocks(17, *first)
    i2, c2 = _lib.traj_list_philox_blocks(17, *second)
    assert i1 == i2 == 17 + 4 * 2 ** 32 and len(c1) == len(c2) == _lib.TRAJ_VERTS
    if sum(first) != sum(second):
        assert not set(c1) & set(c2)
    else:
        assert c1 == c2
    assert i1 >> 32 not in (_lib.ZTASK_PLANE_RESET >> 32, _lib.ZTASK_PLANE_STRIKE >> 32, _lib.ZTASK_PLANE_RESET_TASK >> 32,
                            _lib.ZTASK_PLANE_UPDATE_TASK >> 32)


class _Flags(types.SimpleNamespace):
    pass


def _mixin_task(**over):
    from pulse_b200.terrain_reset import HumanoidPedestrianTerrainResetB200Mixin
    from tests.ztask_standin import StandInZTask

    class Task(HumanoidPedestrianTerrainResetB200Mixin, StandInZTask):
        pass

    t = Task("speed", types.SimpleNamespace(gts=None, _sampling_batch_prob=None), "cpu", 8)
    t.big_ankle, t.real_mesh = False, False
    t.cfg = {"env": {"terrain": {"terrainType": "trimesh"}}}
    t.terrain = types.SimpleNamespace()
    for k, v in over.items():
        setattr(t, k, v)
    return t


@pytest.mark.parametrize("change,words", [
    (lambda t: setattr(t, "humanoid_type", "smplx"), "humanoid_type"),
    (lambda t: t.humanoid_shapes.__setitem__((3, 2), 0.5), "shape variation"),
    (lambda t: setattr(t, "big_ankle", True), "big_ankle"),
    (lambda t: setattr(t, "real_mesh", True), "mesh terrain"),
    (lambda t: setattr(t, "_key_body_ids", torch.tensor([7, 3, 22, 18])), "keyBodies"),
])
def test_mixin_refuses_what_the_device_reset_does_not_serve(change, words):
    from pulse_b200 import _lib
    t = _mixin_task()
    change(t)
    with pytest.raises(_lib.PulseError, match=words):
        t._pulse_terrain_reset_setup()


@pytest.mark.parametrize("flag", ["fixed", "server_mode"])
def test_mixin_refuses_fixed_and_server_mode(monkeypatch, flag):
    from pulse_b200 import _lib, flags_compat
    monkeypatch.setattr(flags_compat, "reference_flags", lambda: _Flags(**{flag: True}))
    with pytest.raises(_lib.PulseError, match=f"flags.{flag}"):
        _mixin_task()._pulse_terrain_reset_setup()


@pytest.mark.parametrize("ttype", ["plane", "none"])
def test_plane_and_none_terrain_are_refused(ttype):
    from pulse_b200 import _lib
    from pulse_b200.terrain_reset import TerrainResetB200
    with pytest.raises(_lib.PulseError, match="walkable table"):
        TerrainResetB200.from_reference(None, None, None, ttype)


def test_mixin_default_state_init_goes_to_the_reference():
    t = _mixin_task()
    t._state_init = types.SimpleNamespace(name="Default")
    with pytest.raises(AssertionError, match="reference reset path"):
        t._reset_envs(torch.arange(3))
