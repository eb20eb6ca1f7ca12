"""Mesh distances without a GPU: the C ABI's entry points, workspace sizes and argument errors, a compile check that the kernels of
csrc/mesh_distance.cu (its own and those of csrc/mesh_csr.cuh it launches) exist and do not spill, and the closest-point formula, pseudonormals and samples of oracle/mesh_distance.py on cases
worked by hand."""
import ctypes
import math
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from oracle import mesh_distance as MD
from permuto_sdf_b200 import _lib
from permuto_sdf_b200.mesh import Mesh, mesh_distance

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ENTRY_POINTS = ("psdf_mesh_closest_points", "psdf_mesh_pseudonormals_workspace_bytes", "psdf_mesh_pseudonormals",
                "psdf_mesh_signed_distance", "psdf_mesh_sample_surface")
KERNELS = ("k_mesh_check<PnWs>", "k_mesh_degree<PnWs>", "k_mesh_scan_tiles<Count, int>", "k_mesh_scan_top", "k_mesh_scan_out<Count, int>",
           "k_mesh_fill<PnWs>", "k_mesh_sort<PnWs>", "k_md_closest", "k_md_sign", "k_md_face_n", "k_md_vert_n", "k_md_edge_n", "k_md_sample")


# ------------------------------------------------------------------------------------------------ C ABI
def test_abi_declares_and_exports_the_entry_points():
    assert set(ENTRY_POINTS) <= set(_lib.declared_symbols())
    ret, args = _lib.PROTOS["psdf_mesh_closest_points"]
    assert ret == "int" and [a for a, _ in args] == ["V", "F", "P", "points", "verts", "faces", "workspace", "dist2_out", "face_out",
                                                     "bary_out", "stream"]
    assert dict(args)["P"] == "long long"
    ret, args = _lib.PROTOS["psdf_mesh_pseudonormals"]
    assert [a for a, _ in args] == ["V", "F", "verts", "faces", "workspace", "face_n", "vert_n", "edge_n", "stream"]
    ret, args = _lib.PROTOS["psdf_mesh_sample_surface"]
    assert [a for a, _ in args] == ["V", "F", "verts", "faces", "cdf", "N", "seed", "points_out", "face_out", "stream"]
    assert dict(args)["cdf"] == "ptr:double" and dict(args)["seed"] == "uint64_t" and dict(args)["N"] == "long long"
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python __graft_entry__.py"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in ENTRY_POINTS:
        assert hasattr(lib, s), "library does not export " + s


@pytest.mark.parametrize("V,F", [(0, 0), (3, 1), (1000, 1999), (12345, 256 * 77 + 1), (2 ** 31 - 1, 2 ** 31 - 1)])
def test_pseudonormal_workspace_sizes(V, F):
    a = lambda n: (n + 255) // 256 * 256
    tiles = (V + 2047) // 2048 + 1
    assert _lib.load_library().psdf_mesh_pseudonormals_workspace_bytes(V, F) == a(256) + a(8 * (V + 1)) + a(4 * V) + a(12 * F) + a(8 * tiles)


def test_argument_errors():
    lib = _lib.load_library()
    ws = lib.psdf_mesh_pseudonormals_workspace_bytes
    assert ws(2 ** 31, 1) == -3 and ws(1, 2 ** 31) == -3 and ws(-1, 0) == -1 and ws(0, -1) == -1
    cp = lib.psdf_mesh_closest_points
    assert cp(3, 1, -1, 8, 8, 8, 8, 8, 8, 8, None) == -1
    assert cp(3, 1, 5, None, 8, 8, 8, 8, 8, 8, None) == -1                # points missing
    assert cp(3, 1, 5, 8, 8, None, 8, 8, 8, 8, None) == -1                # faces missing
    assert cp(3, 1, 5, 8, 8, 8, None, 8, 8, 8, None) == -1                # workspace missing
    assert cp(3, 1, 5, 8, 8, 8, 8, 8, None, 8, None) == -1                # face_out missing
    assert cp(3, 1, 256 * (2 ** 31 - 1) + 1, 8, 8, 8, 8, 8, 8, 8, None) == -3
    assert cp(3, 1, 0, None, 8, 8, 8, None, None, None, None) == 0        # nothing to do, nothing launched
    pn = lib.psdf_mesh_pseudonormals
    assert pn(-1, 0, None, None, 8, None, None, None, None) == -1
    assert pn(3, 1, 8, 8, None, 8, 8, 8, None) == -1                      # workspace missing
    assert pn(3, 1, 8, 8, 8, 8, 8, None, None) == -1                      # edge_n missing
    sd = lib.psdf_mesh_signed_distance
    assert sd(3, 1, 4, 8, 8, 8, 8, 8, None, 8, 8, 8, 8, 8, None) == -1    # vert_n missing
    assert sd(3, 1, 4, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, None, None) == -1    # sdf_out missing
    assert sd(3, 1, 256 * (2 ** 31 - 1) + 1, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, None) == -3
    assert sd(3, 1, 0, None, 8, 8, 8, 8, 8, 8, None, None, None, None, None) == 0
    ss = lib.psdf_mesh_sample_surface
    assert ss(3, 0, 8, 8, 8, 5, 0, 8, 8, None) == -1                      # no face to sample
    assert ss(3, 1, 8, 8, None, 5, 0, 8, 8, None) == -1                   # cdf missing
    assert ss(3, 1, 8, 8, 8, -1, 0, 8, 8, None) == -1
    assert ss(3, 1, 8, 8, 8, 256 * (2 ** 31 - 1) + 1, 0, 8, 8, None) == -3
    assert ss(3, 0, None, None, None, 0, 0, None, None, None) == 0


def test_python_argument_checks():
    m = Mesh(torch.zeros(3, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.closest_points(torch.zeros(1, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.signed_distance(torch.zeros(1, 3))
    with pytest.raises(RuntimeError, match="must be a Mesh"):
        mesh_distance(m, "not a mesh")
    with pytest.raises(RuntimeError, match="CUDA"):
        mesh_distance(m, m)
    with pytest.raises(RuntimeError, match="nr_samples"):
        mesh_distance(m, m, nr_samples=0)
    with pytest.raises(RuntimeError, match="seed"):
        mesh_distance(m, m, seed=-1)


# ------------------------------------------------------------------------------------------------ compile check
@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {r["kernel"]: r for r in wgmma_report.report(("mesh_distance.cu",))}


def test_kernels_and_the_shared_csr_fill_are_built_and_do_not_spill(kernels):
    md = {k: r for k, r in kernels.items() if k.startswith(("k_md_", "k_mesh_"))}
    assert set(md) == set(KERNELS)
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in md.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling


# ------------------------------------------------------------------------------------------------ the oracle's formula by hand
T = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)


def closest1(p, tri=T):
    d2, w = MD.closest_on_triangle(np.array(p, np.float32), tri[0], tri[1], tri[2])
    return float(d2), w.tolist()


def test_interior_edge_and_vertex():
    assert closest1([0.25, 0.25, 2]) == (4.0, [0.5, 0.25, 0.25])                      # over the interior
    assert closest1([0.25, 0.25, -0.5]) == (0.25, [0.5, 0.25, 0.25])                  # under it
    assert closest1([0.5, -1, 0]) == (1.0, [0.5, 0.5, 0.0])                           # beside edge ab
    assert closest1([-2, 0.75, 0]) == (4.0, [0.25, 0.0, 0.75])                        # beside edge ac
    d2, w = closest1([1, 1, 0])                                                        # beside edge bc, at its midpoint
    assert d2 == 0.5 and w == [0.0, 0.5, 0.5]
    assert closest1([-1, -1, 1]) == (3.0, [1.0, 0.0, 0.0])                            # beyond vertex a
    assert closest1([3, -1, 0]) == (5.0, [0.0, 1.0, 0.0])                             # beyond vertex b
    assert closest1([0, 2, 2]) == (5.0, [0.0, 0.0, 1.0])                              # beyond vertex c
    for k in range(3):                                                                 # on the corners themselves
        d2, w = closest1(T[k])
        assert d2 == 0 and w == np.eye(3)[k].tolist()


def test_zero_area_faces_are_their_edges():
    # collinear, c between a and b: a point beside the segment projects onto it
    tri = np.array([[0, 0, 0], [2, 0, 0], [1, 0, 0]], np.float32)
    d2, w = closest1([0.5, 1, 0], tri)
    assert d2 == 1.0 and np.allclose(np.array(w) @ tri, [0.5, 0, 0])
    d2, w = closest1([3, 0, 1], tri)                                                   # beyond the far end b
    assert d2 == 2.0 and np.allclose(np.array(w) @ tri, [2, 0, 0])
    # two corners at one position (distinct indices): the segment between the two positions
    tri = np.array([[0, 0, 0], [0, 0, 0], [0, 4, 0]], np.float32)
    d2, w = closest1([1, 3, 0], tri)
    assert d2 == 1.0 and np.allclose(np.array(w) @ tri, [0, 3, 0])
    # all three at one point
    d2, w = closest1([1, 2, 2], np.zeros((3, 3), np.float32))
    assert d2 == 9.0 and all(math.isfinite(x) for x in w)


def test_brute_force_rules():
    # two copies of one triangle and a face that repeats a vertex: ties go to the smaller index, the repeated face is never taken
    V = np.concatenate([T, T, [[0.25, 0.25, 0.1]]]).astype(np.float32)
    F = np.array([[6, 6, 0], [3, 4, 5], [0, 1, 2]])
    d2, face, bary = MD.closest_points(V, F, np.array([[0.25, 0.25, 0.1], [0.25, 0.25, 1.0]], np.float32))
    assert face.tolist() == [1, 1] and d2.tolist() == [np.float32(0.1) ** 2, 1.0]
    # no valid face
    d2, face, bary = MD.closest_points(V, np.array([[0, 0, 1]]), np.zeros((2, 3), np.float32))
    assert np.isinf(d2).all() and (face == -1).all() and (bary == 0).all()
    d2, face, _ = MD.closest_points(V, np.zeros((0, 3), int), np.zeros((1, 3), np.float32))
    assert np.isinf(d2).all() and (face == -1).all()


def test_pseudonormals_of_a_tetrahedron_and_the_sign():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    F = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])                         # outward
    fn, vn, en = MD.pseudonormals(V, F)
    assert np.allclose(fn[0], [0, 0, -1]) and np.allclose(fn[3], np.ones(3) / math.sqrt(3))
    assert np.allclose(vn[0] / np.linalg.norm(vn[0]), -np.ones(3) / math.sqrt(3))      # the corner at the origin points out along -1
    assert np.allclose(en[0, 0], fn[0] + fn[2])                                         # edge 0 -> 2 is shared by faces 0 and 2
    P = np.array([[0.1, 0.1, 0.1], [-1, -1, -1], [0.5, 0.5, 0.5], [0.2, 0.2, -0.3], [0.5, -0.2, -0.2]], np.float32)
    _, face, bary = MD.closest_points(V, F, P)
    s = MD.signed_cos(V, F, P, face, bary)
    assert (np.sign(s) == [-1, 1, 1, 1, 1]).all()


def test_samples():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5], [5, 5, 5], [5, 5, 5], [0, 0, 1]], np.float32)
    F = np.array([[0, 1, 2], [3, 4, 5], [0, 1, 6]])
    area = np.array([0.5, 0.0, 0.5])
    pts, face = MD.sample_surface(V, F, np.cumsum(area), 20000, 7)
    assert set(face.tolist()) == {0, 2} and abs((face == 0).mean() - 0.5) < 0.02
    # every sample lies on its face; the first N of a larger draw are the smaller draw
    assert (pts[face == 0][:, 2] == 0).all() and (pts[face == 2][:, 1] == 0).all()
    assert (pts[:, :2] >= 0).all() and (pts.sum(1) <= 1 + 1e-6).all()
    p2, f2 = MD.sample_surface(V, F, np.cumsum(area), 100, 7)
    assert np.array_equal(p2, pts[:100]) and np.array_equal(f2, face[:100])
    # the generator is SplitMix64: its first output for seed 0 (Vigna's reference implementation)
    assert int(MD.splitmix64(0, 0)) == 0xE220A8397B1DCDAF


def test_fp64_distance_of_the_oracle():
    d = MD.point_mesh_distance64(T, np.array([[0, 1, 2]]), np.array([[0.25, 0.25, 2], [0.5, -1, 0], [-1, -1, 1]]))
    assert np.allclose(d, [2, 1, math.sqrt(3)], rtol=0, atol=1e-12)
