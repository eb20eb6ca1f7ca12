"""Mesh ray casting without a GPU: the C ABI's entry points, workspace sizes and argument errors, a compile check that the BVH build
kernels of csrc/mesh_bvh.cu (its own and those of csrc/mesh_csr.cuh it launches) and the any-hit kernels of csrc/mesh_raycast.cu exist and
do not spill, the ray-triangle test of oracle/raycast.py on cases worked by hand, and the file selection of load_mesh_sequence."""
import ctypes
import math
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from oracle import raycast as RC
from permuto_sdf_b200 import _lib
from permuto_sdf_b200.mesh import Mesh, fibonacci_directions, natural_key, sequence_files

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ENTRY_POINTS = ("psdf_mesh_bvh_workspace_bytes", "psdf_mesh_bvh_build", "psdf_mesh_occluded", "psdf_mesh_ambient_occlusion")
# the build, compiled from csrc/mesh_bvh.cu, and the any-hit queries, compiled from csrc/mesh_raycast.cu
BUILD_KERNELS = ("k_mesh_check<Ws>", "k_mesh_scan_tiles<Count, int>", "k_mesh_scan_top", "k_mesh_scan_out<Count, int>", "k_bvh_bounds",
                 "k_bvh_morton", "k_bvh_hist", "k_bvh_scatter", "k_bvh_internal", "k_bvh_leaves")
QUERY_KERNELS = ("k_rc_occluded", "k_rc_ao", "k_rc_vis")


# ------------------------------------------------------------------------------------------------ C ABI
def _size(V, F):
    a = lambda n: (n + 255) // 256 * 256
    nh = 256 * ((F + 255) // 256)
    tiles = (nh + 2047) // 2048 + 1
    return (a(256) + a(32) + 4 * a(4 * F) + a(4 * nh) + a(8 * (nh + 1)) + a(8 * tiles) + a(64 * max(F - 1, 0)) + a(4 * max(2 * F - 1, 0))
            + a(4 * max(F - 1, 0)) + a(48 * F) + a(4 * V))


def test_abi_declares_and_exports_the_entry_points():
    assert set(ENTRY_POINTS) <= set(_lib.declared_symbols())
    ret, args = _lib.PROTOS["psdf_mesh_occluded"]
    assert ret == "int" and [a for a, _ in args] == ["V", "F", "R", "origins", "dirs", "tnear", "tfar", "workspace", "hit_out", "stream"]
    assert dict(args)["R"] == "long long"
    ret, args = _lib.PROTOS["psdf_mesh_ambient_occlusion"]
    assert [a for a, _ in args] == ["V", "F", "S", "verts", "normals", "dirs", "workspace", "vis_out", "stream"]
    assert _lib.PROTOS["psdf_mesh_bvh_workspace_bytes"][0] == "long long"
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python __graft_entry__.py"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in ENTRY_POINTS:
        assert hasattr(lib, s), "library does not export " + s


@pytest.mark.parametrize("V,F", [(0, 0), (3, 1), (5, 2), (1000, 1999), (12345, 256 * 77 + 1), (2 ** 31 - 1, 2 ** 31 - 1)])
def test_workspace_sizes(V, F):
    assert _lib.load_library().psdf_mesh_bvh_workspace_bytes(V, F) == _size(V, F)


def test_workspace_limits_and_argument_errors():
    lib = _lib.load_library()
    ws = lib.psdf_mesh_bvh_workspace_bytes
    assert ws(2 ** 31, 1) == -3 and ws(1, 2 ** 31) == -3
    assert ws(-1, 0) == -1 and ws(0, -1) == -1
    assert lib.psdf_mesh_bvh_build(-1, 0, None, None, 8, None) == -1
    assert lib.psdf_mesh_bvh_build(3, 1, 8, None, 8, None) == -1                        # faces missing
    assert lib.psdf_mesh_bvh_build(3, 1, 8, 8, None, None) == -1                        # workspace missing
    assert lib.psdf_mesh_occluded(3, 1, -1, 8, 8, 0.0, 1.0, 8, 8, None) == -1
    assert lib.psdf_mesh_occluded(3, 1, 5, None, 8, 0.0, 1.0, 8, 8, None) == -1         # origins missing
    assert lib.psdf_mesh_occluded(3, 1, 5, 8, 8, 0.0, 1.0, 8, None, None) == -1         # hit_out missing
    assert lib.psdf_mesh_occluded(3, 1, 256 * (2 ** 31 - 1) + 1, 8, 8, 0.0, 1.0, 8, 8, None) == -3
    assert lib.psdf_mesh_occluded(3, 1, 0, None, None, 0.0, 1.0, 8, None, None) == 0    # nothing to do, nothing launched
    assert lib.psdf_mesh_ambient_occlusion(3, 1, 0, 8, 8, 8, 8, 8, None) == -1          # S < 1
    assert lib.psdf_mesh_ambient_occlusion(3, 1, 4, 8, None, 8, 8, 8, None) == -1       # normals missing
    assert lib.psdf_mesh_ambient_occlusion(2 ** 30, 1, 2 ** 10, 8, 8, 8, 8, 8, None) == -3


def test_python_argument_checks():
    m = Mesh(torch.zeros(3, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    with pytest.raises(RuntimeError, match="recalculate_normals"):
        m.ambient_occlusion(100)
    with pytest.raises(RuntimeError, match="nr_samples"):
        m.ambient_occlusion(0)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.occluded(torch.zeros(1, 3), torch.ones(1, 3))
    other = Mesh(torch.zeros(3, 3), torch.tensor([[0, 2, 1]], dtype=torch.int32))
    with pytest.raises(RuntimeError, match="different faces"):
        m.interpolate(other, 0.5)
    with pytest.raises(RuntimeError, match="shape"):
        m.interpolate(Mesh(torch.zeros(4, 3), m.F), 0.5)
    V2 = torch.randn(3, 3)
    r = m.interpolate(Mesh(V2, m.F.clone()), 0.3)
    assert torch.equal(r.V, torch.lerp(m.V, V2, 0.3)) and torch.equal(r.F, m.F) and r.F is not m.F and r.NV is None


# ------------------------------------------------------------------------------------------------ compile check
@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {(r["unit"], r["kernel"]): r for r in wgmma_report.report(("mesh_bvh.cu", "mesh_raycast.cu"))}


def test_build_and_query_kernels_are_built_and_do_not_spill(kernels):
    units = {"mesh_bvh.cu": (("k_bvh_", "k_rc_", "k_mesh_"), BUILD_KERNELS),
             "mesh_raycast.cu": (("k_bvh_", "k_rc_"), QUERY_KERNELS)}       # it also emits mesh_csr.cuh's k_mesh_scan_top, never launched
    for unit, (prefixes, expected) in units.items():
        rc = {k: r for (u, k), r in kernels.items() if u == unit and k.startswith(prefixes)}
        assert set(rc) == set(expected), unit
        spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in rc.items() if r["spill_st"] or r["spill_ld"]}
        assert not spilling, (unit, spilling)


# ------------------------------------------------------------------------------------------------ the oracle's test by hand
T = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)


def hit1(o, d, tnear=0.0, tfar=math.inf, tri=T):
    return bool(RC.hit(tri[0], tri[1], tri[2], np.array(o, np.float32), np.array(d, np.float32), tnear, tfar))


def test_interior_edge_and_vertex():
    assert hit1([0.25, 0.25, 1], [0, 0, -1])
    assert hit1([0.5, 0, 1], [0, 0, -1]) and hit1([0.5, 0.5, 1], [0, 0, -1]) and hit1([0, 0.5, 1], [0, 0, -1])     # edges
    assert hit1([0, 0, 1], [0, 0, -1]) and hit1([1, 0, 1], [0, 0, -1]) and hit1([0, 1, 1], [0, 0, -1])             # vertices
    assert not hit1([0.6, 0.6, 1], [0, 0, -1]) and not hit1([-0.01, 0.2, 1], [0, 0, -1])
    assert not hit1([0.25, 0.25, 1], [0, 0, 1])                                                                     # behind the origin


def test_back_faces_are_hit():
    assert hit1([0.25, 0.25, -1], [0, 0, 1]) and hit1([0.25, 0.25, 1], [0, 0, -1])


def test_t_at_the_interval_ends():
    # t = 1 exactly: open at both ends
    assert not hit1([0.25, 0.25, 1], [0, 0, -1], tnear=1.0) and hit1([0.25, 0.25, 1], [0, 0, -1], tnear=np.nextafter(np.float32(1), 0))
    assert not hit1([0.25, 0.25, 1], [0, 0, -1], tfar=1.0) and hit1([0.25, 0.25, 1], [0, 0, -1], tfar=np.nextafter(np.float32(1), 2))
    # an origin on the triangle: t = 0, which tnear = 1e-4 excludes
    assert not hit1([0.25, 0.25, 0], [0, 0, 1], tnear=1e-4) and hit1([0.25, 0.25, 0], [0, 0, 1], tnear=-1.0)


def test_parallel_rays_have_det_zero():
    assert not hit1([0.25, 0.25, 0], [1, 0, 0], tnear=-1.0)          # in the plane: det == 0
    assert not hit1([0.25, 0.25, 1], [1, 1, 0])


def test_degenerate_triangles_are_never_hit():
    for tri in (np.array([[0, 0, 0], [0, 0, 0], [1, 1, 0]], np.float32), np.array([[0, 0, 0], [1, 1, 0], [2, 2, 0]], np.float32),
                np.zeros((3, 3), np.float32)):
        assert not hit1([0.5, 0.5, 1], [0, 0, -1], tri=tri) and not hit1([0, 0, 1], [0, 0, -1], tri=tri)


def test_occluded_and_ambient_occlusion_of_the_oracle():
    V = np.concatenate([T, T + np.float32([0, 0, 2])])
    F = np.array([[0, 1, 2], [3, 4, 5]])
    o = np.array([[0.2, 0.2, 1], [0.2, 0.2, 1], [3, 3, 1]], np.float32)
    d = np.array([[0, 0, 1], [0, 0, -1], [0, 0, 1]], np.float32)
    assert RC.occluded(V, F, o, d).tolist() == [True, True, False]
    assert not RC.occluded(V, np.zeros((0, 3), int), o, d).any()
    # a lone triangle: a vertex sees everything except along its own plane (det == 0), so vis = 1
    NV = np.tile(np.float32([0, 0, 1]), (3, 1))
    assert (RC.ambient_occlusion(T, np.array([[0, 1, 2]]), NV, 64) == 1).all()


def test_fibonacci_directions():
    D = fibonacci_directions(100)
    assert D.dtype == np.float32 and D.shape == (100, 3)
    assert np.array_equal(D, RC.directions(100))
    assert np.allclose(np.linalg.norm(D.astype(np.float64), axis=1), 1, atol=1e-6)
    assert abs(float(D[:, 2].astype(np.float64).mean())) < 1e-6 and D[0, 2] == np.float32(1 - 1 / 100)


# ------------------------------------------------------------------------------------------------ load_mesh_sequence's file selection
def test_natural_sort_key():
    names = ["f_10.obj", "f_2.obj", "f_1.obj", "f_100.ply", "g_0.obj", "f_9.obj"]
    assert sorted(names, key=natural_key) == ["f_1.obj", "f_2.obj", "f_9.obj", "f_10.obj", "f_100.ply", "g_0.obj"]
    assert sorted(["a10b2", "a10b10", "a9b100"], key=natural_key) == ["a9b100", "a10b2", "a10b10"]


def test_file_selection():
    names = ["frame_%d.obj" % i for i in range(14)] + ["notes.txt", "frame_3.stl", "script.py"]
    sel = sequence_files(names)
    assert sel == ["frame_%d.obj" % i for i in range(13)]                      # 14 files give 13: i > min(12, n) breaks
    assert sequence_files(["b_2.ply", "b_10.ply", "b_1.obj"]) == ["b_1.obj", "b_2.ply", "b_10.ply"]
    assert sequence_files(["x_%d.ply" % i for i in range(12)]) == ["x_%d.ply" % i for i in range(12)]
    assert sequence_files(["x_%d.ply" % i for i in range(13)]) == ["x_%d.ply" % i for i in range(13)]
    assert sequence_files(["only.obj", "a.txt"]) == ["only.obj"]


def test_fewer_than_two_frames_are_refused(tmp_path):
    from permuto_sdf_b200.mesh import load_mesh_sequence
    (tmp_path / "a_0.obj").write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n")
    with pytest.raises(RuntimeError, match="at least 2"):
        load_mesh_sequence(tmp_path, device="cpu")
