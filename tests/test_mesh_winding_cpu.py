"""Winding numbers without a GPU: the C ABI's entry points, workspace sizes and argument errors, the Python argument checks, a compile
check that the kernels of csrc/mesh_winding.cu exist and do not spill, and the fp64 oracle (oracle/winding.py) on cases worked by hand."""
import ctypes
import math
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from oracle import winding as WN
from permuto_sdf_b200 import _lib
from permuto_sdf_b200.mesh import Mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ENTRY_POINTS = ("psdf_mesh_winding_workspace_bytes", "psdf_mesh_winding_build", "psdf_mesh_winding_number")
KERNELS = ("k_wn_build", "k_wn_query")


# ------------------------------------------------------------------------------------------------ meshes worked by hand
TET_V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
TET_F = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)          # outward


def uv_sphere(n_lat, n_lon, centre=(0.0, 0.0, 0.0), radius=1.0, hemisphere=False):
    """a latitude-longitude sphere with outward faces; hemisphere=True keeps the upper half, its rim on the plane z = centre z, open"""
    rings = n_lat if hemisphere else n_lat - 1
    th = np.arange(1, rings + 1) * ((math.pi / 2 if hemisphere else math.pi) / n_lat)
    ph = np.arange(n_lon) * (2 * math.pi / n_lon)
    ring = np.stack([np.sin(th)[:, None] * np.cos(ph), np.sin(th)[:, None] * np.sin(ph), np.cos(th)[:, None] + 0 * ph], -1).reshape(-1, 3)
    if hemisphere:
        ring[-n_lon:, 2] = 0.0                                 # the rim exactly on the equator
    V = np.concatenate([[[0, 0, 1]], ring] + ([] if hemisphere else [[[0, 0, -1]]]))
    F = []
    r = lambda i, j: 1 + i * n_lon + j % n_lon
    for j in range(n_lon):
        F.append([0, r(0, j), r(0, j + 1)])
        for i in range(rings - 1):
            F += [[r(i, j), r(i + 1, j), r(i + 1, j + 1)], [r(i, j), r(i + 1, j + 1), r(i, j + 1)]]
        if not hemisphere:
            F.append([len(V) - 1, r(rings - 1, j + 1), r(rings - 1, j)])
    return (V * radius + np.asarray(centre)).astype(np.float32), np.asarray(F, np.int32)


# ------------------------------------------------------------------------------------------------ C ABI
def test_abi_declares_and_exports_the_entry_points():
    assert set(ENTRY_POINTS) <= set(_lib.declared_symbols())
    ret, args = _lib.PROTOS["psdf_mesh_winding_workspace_bytes"]
    assert ret == "long long" and args == [("nr_vertices", "long long"), ("nr_faces", "long long")]
    ret, args = _lib.PROTOS["psdf_mesh_winding_build"]
    assert ret == "int" and [a for a, _ in args] == ["V", "F", "verts", "faces", "bvh_workspace", "workspace", "stream"]
    assert dict(args)["bvh_workspace"] == "ptr:uint8_t" and dict(args)["workspace"] == "ptr:uint8_t"
    ret, args = _lib.PROTOS["psdf_mesh_winding_number"]
    assert ret == "int" and [a for a, _ in args] == ["V", "F", "P", "points", "bvh_workspace", "workspace", "beta", "w_out", "stream"]
    assert dict(args)["P"] == "long long" and dict(args)["beta"] == "float" and dict(args)["w_out"] == "ptr:float"
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python __graft_entry__.py"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in ENTRY_POINTS:
        assert hasattr(lib, s), "library does not export " + s


@pytest.mark.parametrize("V,F", [(0, 0), (3, 1), (4, 2), (1000, 1999), (2 ** 31 - 1, 2 ** 31 - 1)])
def test_workspace_sizes(V, F):
    a = lambda n: (n + 255) // 256 * 256
    n = max(F - 1, 0)
    assert _lib.load_library().psdf_mesh_winding_workspace_bytes(V, F) == a(144 * n) + a(4 * n)


def test_argument_errors():
    lib = _lib.load_library()
    ws = lib.psdf_mesh_winding_workspace_bytes
    assert ws(2 ** 31, 1) == -3 and ws(1, 2 ** 31) == -3 and ws(-1, 0) == -1 and ws(0, -1) == -1
    b = lib.psdf_mesh_winding_build
    assert b(-1, 0, None, None, 8, 8, None) == -1
    assert b(3, -1, 8, 8, 8, 8, None) == -1
    assert b(3, 2, 8, 8, None, 8, None) == -1                               # BVH workspace missing
    assert b(3, 2, 8, 8, 8, None, None) == -1                               # workspace missing with an internal node
    assert b(3, 1, None, None, 8, None, None) == 0                          # F = 1: no internal node, nothing launched
    assert b(0, 0, None, None, 8, None, None) == 0
    wn = lib.psdf_mesh_winding_number
    inf = float("inf")
    assert wn(3, 2, -1, 8, 8, 8, ctypes.c_float(2.0), 8, None) == -1
    assert wn(3, 2, 5, None, 8, 8, ctypes.c_float(2.0), 8, None) == -1     # points missing
    assert wn(3, 2, 5, 8, None, 8, ctypes.c_float(2.0), 8, None) == -1     # BVH workspace missing
    assert wn(3, 2, 5, 8, 8, None, ctypes.c_float(2.0), 8, None) == -1     # workspace missing
    assert wn(3, 2, 5, 8, 8, 8, ctypes.c_float(2.0), None, None) == -1     # w_out missing
    for beta in (0.0, -1.0, -inf, float("nan")):
        assert wn(3, 2, 5, 8, 8, 8, ctypes.c_float(beta), 8, None) == -1
    assert wn(3, 2, 256 * (2 ** 31 - 1) + 1, 8, 8, 8, ctypes.c_float(2.0), 8, None) == -3
    assert wn(3, 2, 256 * (2 ** 31 - 1) + 1, 8, 8, 8, ctypes.c_float(inf), 8, None) == -3
    assert wn(3, 2, 0, None, 8, 8, ctypes.c_float(2.0), None, None) == 0    # nothing to do, nothing launched


def test_python_argument_checks():
    m = Mesh(torch.zeros(3, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.winding_number(torch.zeros(1, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.signed_distance(torch.zeros(1, 3), sign="winding")
    for beta in (0, 0.0, -1.0, math.nan, -math.inf, True, "2"):
        with pytest.raises(RuntimeError, match="beta must be a positive number"):
            m.winding_number(torch.zeros(1, 3), beta=beta)
    with pytest.raises(RuntimeError, match="unknown sign 'parity'"):
        m.signed_distance(torch.zeros(1, 3), sign="parity")


# ------------------------------------------------------------------------------------------------ compile check
@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {r["kernel"]: r for r in wgmma_report.report(("mesh_winding.cu",))}


def test_kernels_are_built_and_do_not_spill(kernels):
    wn = {k: r for k, r in kernels.items() if k.startswith("k_wn_")}
    assert set(wn) == set(KERNELS)
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in wn.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling


# ------------------------------------------------------------------------------------------------ the oracle by hand
def test_tetrahedron_inside_outside_and_flipped():
    inside = np.array([[0.1, 0.1, 0.1], [0.2, 0.3, 0.4], [0.01, 0.01, 0.97]], np.float32)
    outside = np.array([[2, 2, 2], [-0.1, 0.2, 0.2], [0.5, 0.5, 0.5], [-5, 3, 1]], np.float32)
    w = WN.winding_numbers(TET_V, TET_F, np.concatenate([inside, outside]))
    assert np.abs(w[:3] - 1).max() < 1e-14 and np.abs(w[3:]).max() < 1e-14
    wf = WN.winding_numbers(TET_V, TET_F[:, ::-1], inside)
    assert np.abs(wf + 1).max() < 1e-14


def test_single_triangle_seen_from_its_normal_axis():
    """the triangle x + y + z = 1 of the positive octant covers the octant seen from the origin: a solid angle of 4 pi / 8, so w = 1/8;
    its mirror point (2/3, 2/3, 2/3) on the axis sees the back, -1/8; the same for every triangle x + y + z = s, s > 0"""
    for s in (1.0, 0.25, 8.0):
        V = np.eye(3, dtype=np.float32) * np.float32(s)
        w = WN.winding_numbers(V, [[0, 1, 2]], np.array([[0, 0, 0], [2 * s / 3] * 3], np.float32))
        assert abs(w[0] - 0.125) < 1e-14 and abs(w[1] + 0.125) < 1e-7      # (2 s / 3 rounds to fp32)


def test_hemisphere_from_its_centre_is_one_half():
    """the rim lies on z = 0, so from the centre every rim edge projects onto the equator and the cap covers exactly the upper half"""
    V, F = uv_sphere(8, 24, hemisphere=True)
    w = WN.winding_numbers(V, F, np.zeros((1, 3), np.float32))
    assert abs(w[0] - 0.5) < 1e-13
    assert abs(WN.winding_numbers(V, F[:, ::-1], np.zeros((1, 3), np.float32))[0] + 0.5) < 1e-13


def test_two_overlapping_spheres_give_two_in_the_overlap():
    a = uv_sphere(16, 32, (-0.5, 0, 0))
    b = uv_sphere(16, 32, (0.5, 0, 0))
    V = np.concatenate([a[0], b[0]])
    F = np.concatenate([a[1], b[1] + len(a[0])])
    P = np.array([[0, 0, 0], [0.1, 0.1, -0.1], [-1.2, 0, 0], [1.2, 0.1, 0], [3, 0, 0], [0, 2, 0]], np.float32)
    w = WN.winding_numbers(V, F, P)
    assert np.abs(w - [2, 2, 1, 1, 0, 0]).max() < 1e-12


def test_degenerate_faces_contribute_nothing():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [0, 0, 0]], np.float32)
    P = np.array([[0.2, 0.2, 0.0], [3, 3, 0], [0, 0, 0], [0.2, 0.2, 1.0]], np.float32)
    # p in the face's plane (inside it, outside it) and p on a corner: det == 0
    assert (WN.winding_numbers(V, [[0, 1, 2]], P[:3]) == 0).all()
    assert WN.winding_numbers(V, [[0, 1, 2]], P[3:])[0] < 0              # above a +z face: its back
    # collinear corners (zero area), a repeated vertex index, and two corners equal in value under distinct indices
    for f in ([0, 1, 3], [0, 0, 2], [1, 2, 2], [4, 1, 0], [0, 4, 2]):
        assert (WN.winding_numbers(V, [f], P) == 0).all(), f
    assert (WN.rounding_bound(V, [[0, 0, 2], [0, 4, 2]], P) <= 2.0 ** -140).all()


def test_rounding_bound_is_small_away_from_the_faces_and_covers_the_plane():
    V, F = uv_sphere(12, 24)
    rng = np.random.default_rng(0)
    d = rng.standard_normal((200, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    far = (d * rng.uniform(0.0, 0.8, (200, 1))).astype(np.float32)
    assert WN.rounding_bound(V, F, far).max() < 30 * 2.0 ** -24 * len(F)            # about 20 u per face, worst case summed
    # a point in a face's plane, inside that face: the sign of det is undecided, and the bound allows the whole swing
    tri = V[F[5]].astype(np.float64)
    p = tri.mean(0).astype(np.float32)[None]
    assert WN.rounding_bound(V, F[5:6], p)[0] >= 0.5
