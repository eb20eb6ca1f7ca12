"""Mesh decimation and vertex normals without a GPU: the argument checks of Mesh.decimate and Mesh.recalculate_normals, the C ABI's
entry points and their limits, a compile check that the kernels of csrc/mesh_decimate.cu (its own and those of csrc/mesh_csr.cuh it
launches) exist and do not spill, and the properties of oracle/decimate.py on small marching-cubes meshes."""
import ctypes
import os
import shutil
import sys

import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import decimate as D
from oracle import marching_cubes as MC
from permuto_sdf_b200 import _lib
from permuto_sdf_b200.mesh import Mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ENTRY_POINTS = ("psdf_mesh_decimate_workspace_bytes", "psdf_mesh_normals_workspace_bytes", "psdf_mesh_decimate_begin",
                "psdf_mesh_decimate_round", "psdf_mesh_normals")
KERNELS = ("k_mesh_check<Ws>", "k_mesh_degree<Ws>", "k_mesh_scan_tiles<Count, int>", "k_mesh_scan_tiles<Kept, unsigned char>",
           "k_mesh_scan_top", "k_mesh_scan_out<Count, int>", "k_mesh_scan_out<Kept, unsigned char>", "k_mesh_fill<Ws>", "k_mesh_sort<Ws>",
           "k_dc_lock",
           "k_dc_quadric", "k_dc_key", "k_dc_best2", "k_dc_choose", "k_dc_select", "k_dc_apply", "k_dc_compact", "k_dc_copy", "k_dc_normals")


def tri_mesh(V=None, F=None):
    return Mesh(torch.zeros(3, 3) if V is None else V, torch.tensor([[0, 1, 2]], dtype=torch.int32) if F is None else F)


def both(m):
    return [lambda: m.decimate(0), m.recalculate_normals]


# ------------------------------------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("V", [torch.zeros(3, 3, dtype=torch.float64), torch.zeros(3, 3, dtype=torch.float16), np.zeros((3, 3), np.float32)])
def test_vertices_of_another_dtype_are_refused(V):
    for fn in both(tri_mesh(V=V)):
        with pytest.raises(RuntimeError, match="float32"):
            fn()


@pytest.mark.parametrize("V", [torch.zeros(9), torch.zeros(3, 4), torch.zeros(1, 3, 3)])
def test_vertices_of_another_shape_are_refused(V):
    for fn in both(tri_mesh(V=V)):
        with pytest.raises(RuntimeError, match=r"shape \[V,3\]"):
            fn()


@pytest.mark.parametrize("F", [torch.zeros(1, 3, dtype=torch.int64), torch.zeros(1, 3), np.zeros((1, 3), np.int32)])
def test_faces_of_another_dtype_are_refused(F):
    for fn in both(tri_mesh(F=F)):
        with pytest.raises(RuntimeError, match="int32"):
            fn()


@pytest.mark.parametrize("F", [torch.zeros(6, dtype=torch.int32), torch.zeros(2, 4, dtype=torch.int32)])
def test_faces_of_another_shape_are_refused(F):
    for fn in both(tri_mesh(F=F)):
        with pytest.raises(RuntimeError, match=r"shape \[F,3\]"):
            fn()


def test_cpu_tensors_are_refused():
    for fn in both(tri_mesh()):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn()


@pytest.mark.parametrize("k", [-1, -(2 ** 40), 1.0, 2.5, "3", None, True, False, np.float32(4)])
def test_target_must_be_a_non_negative_integer(k):
    with pytest.raises(RuntimeError, match="nr_target_faces"):
        tri_mesh().decimate(k)


# ------------------------------------------------------------------------------------------------ C ABI
def _sizes(V, F, decimate):
    a = lambda n: (n + 255) // 256 * 256
    tiles = (max(V + 1, F) + 2047) // 2048 + 1
    n = a(256) + a(8 * (V + 1)) + a(4 * V) + a(12 * F) + a(8 * tiles)
    if decimate:
        n += a(80 * V) + 2 * a(8 * V) + a(V) + a(8 * (V // 2 + 1)) + a(24 * F + 8) + a(F)
    return n


def test_abi_declares_and_exports_the_entry_points():
    assert set(ENTRY_POINTS) <= set(_lib.declared_symbols())
    ret, args = _lib.PROTOS["psdf_mesh_decimate_round"]
    assert ret == "int" and [a for a, _ in args] == ["V", "F0", "F", "allowed", "verts", "faces", "workspace", "removed", "stream"]
    assert dict(args)["allowed"] == "long long"
    assert _lib.PROTOS["psdf_mesh_decimate_workspace_bytes"][0] == "long long"
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python __graft_entry__.py"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in ENTRY_POINTS:
        assert hasattr(lib, s), "library does not export " + s


@pytest.mark.parametrize("V,F", [(0, 0), (5, 7), (1000, 1999), (2 ** 31 - 1, 2 ** 31 - 1), (3, 2 ** 31 - 1)])
def test_workspace_sizes(V, F):
    lib = _lib.load_library()
    assert lib.psdf_mesh_decimate_workspace_bytes(V, F) == _sizes(V, F, True)
    assert lib.psdf_mesh_normals_workspace_bytes(V, F) == _sizes(V, F, False)


def test_workspace_limits():
    lib = _lib.load_library()
    for ws in (lib.psdf_mesh_decimate_workspace_bytes, lib.psdf_mesh_normals_workspace_bytes):
        assert ws(2 ** 31, 1) == -3 and ws(1, 2 ** 31) == -3
        assert ws(-1, 0) == -1 and ws(0, -1) == -1


def test_argument_errors_before_any_launch():
    lib = _lib.load_library()
    assert lib.psdf_mesh_decimate_begin(-1, 0, None, None, 8, None, None) == -1
    assert lib.psdf_mesh_decimate_begin(3, 1, 8, None, 8, 8, None) == -1             # faces missing
    assert lib.psdf_mesh_decimate_round(3, 1, 2, 1, 8, 8, 8, 8, None) == -1          # more faces than begin had
    assert lib.psdf_mesh_decimate_round(3, 1, 1, -1, 8, 8, 8, 8, None) == -1         # negative allowed
    assert lib.psdf_mesh_normals(3, 1, 8, 8, None, 8, None) == -1                     # workspace missing


# ------------------------------------------------------------------------------------------------ compile check
@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {r["kernel"]: r for r in wgmma_report.report(("mesh_decimate.cu",))}


def test_kernels_and_the_shared_csr_fill_are_built_and_do_not_spill(kernels):
    dc = {k: r for k, r in kernels.items() if k.startswith(("k_dc_", "k_mesh_"))}
    assert set(dc) == set(KERNELS)
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in dc.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling


# ------------------------------------------------------------------------------------------------ the oracle
@pytest.fixture(scope="module")
def small_meshes():
    return {"sphere": MC.marching_cubes(C.sphere_volume((22,) * 3, (10.3, 10.6, 10.1), 8.0), 0.0),
            "torus": MC.marching_cubes(C.torus_volume((30, 30, 14), (14.4, 14.7, 6.6), 9.0, 4.0), 0.0),
            "random": MC.marching_cubes(C.random_field((24, 24, 24), seed=3), 0.0)}


@pytest.mark.parametrize("name", ["sphere", "torus", "random"])
@pytest.mark.parametrize("frac", [0.5, 0.1, 0.0])
def test_oracle_keeps_topology_and_reaches_the_target(small_meshes, name, frac):
    V, F = small_meshes[name]
    target = int(frac * len(F))
    Vd, Fd, NV, rounds = D.decimate_mesh(V, F, target, True)
    assert rounds > 0
    assert C.closed_and_oriented(Fd, len(Vd))
    assert C.euler_characteristic(Fd) == C.euler_characteristic(F)
    p = Vd.astype(np.float64)[Fd]
    assert (np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1) > 0).all()
    if frac > 0:
        assert len(Fd) in (target, target - 1)
    assert np.allclose(np.linalg.norm(NV, axis=1), 1, atol=1e-5)


def test_oracle_no_op_and_locks(small_meshes):
    V, F = small_meshes["sphere"]
    Vd, Fd, NV, rounds = D.decimate_mesh(V, F, len(F), True)
    assert rounds == 0 and np.array_equal(Vd, V) and np.array_equal(Fd, F) and NV is None
    # an open mesh: every vertex on the cut is locked and keeps its position
    keep = V[:, 0] < 10.0
    new_id = np.cumsum(keep) - 1
    Fo = new_id[F[keep[F].all(1)]]
    Vo = V[keep]
    _, _, _, lock = D.begin(Vo, Fo)
    Vd, Fd, removed, _ = D.decimate(Vo, Fo, 0)
    assert lock.any() and not removed[lock].any()
    assert np.array_equal(Vd[lock], Vo[lock])
