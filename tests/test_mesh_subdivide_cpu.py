"""Mesh subdivision without a GPU: the argument checks of Mesh.upsample, the C ABI's entry points and their limits, a compile check that
the kernels of csrc/mesh_subdivide.cu (its own and those of csrc/mesh_csr.cuh it launches) exist and do not spill, and the properties of
oracle/subdivide.py: counts, Euler characteristic, closed and oriented meshes, exact midpoints, a tetrahedron computed by hand in both
modes, a flat open grid and a non-manifold fan."""
import ctypes
import os
import shutil
import sys

import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import marching_cubes as MC
from oracle import subdivide as S
from permuto_sdf_b200 import _lib
from permuto_sdf_b200.mesh import Mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ENTRY_POINTS = ("psdf_mesh_subdivide_workspace_bytes", "psdf_mesh_subdivide_count", "psdf_mesh_subdivide_emit")
KERNELS = ("k_mesh_check<Ws>", "k_mesh_degree<Ws>", "k_mesh_scan_tiles<Count, int>", "k_mesh_scan_tiles<Owns, int>", "k_mesh_scan_top",
           "k_mesh_scan_out<Count, int>", "k_mesh_scan_out<Owns, int>", "k_sd_fill", "k_sd_edge", "k_sd_sort", "k_sd_even", "k_sd_odd",
           "k_sd_faces")


def tri_mesh(V=None, F=None):
    return Mesh(torch.zeros(3, 3) if V is None else V, torch.tensor([[0, 1, 2]], dtype=torch.int32) if F is None else F)


# ------------------------------------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("k", [-1, 1.0, "2", None, True, np.float32(1)])
def test_rounds_must_be_a_non_negative_integer(k):
    with pytest.raises(RuntimeError, match="nr_subdivisions"):
        tri_mesh().upsample(k, True)


def test_inputs_are_checked_as_decimate_does():
    with pytest.raises(RuntimeError, match="float32"):
        tri_mesh(V=torch.zeros(3, 3, dtype=torch.float64)).upsample(1, True)
    with pytest.raises(RuntimeError, match=r"shape \[F,3\]"):
        tri_mesh(F=torch.zeros(2, 4, dtype=torch.int32)).upsample(1, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        tri_mesh().upsample(1, True)


@pytest.mark.parametrize("nf,rounds", [(2 ** 29, 1), (2 ** 27, 2), (2 ** 20, 6)])
def test_oversized_results_are_refused_from_the_counts(nf, rounds):
    # an expanded view: nothing of the size is allocated, and the count check comes before any other
    Fc = torch.zeros(1, 3, dtype=torch.int32).expand(nf, 3)
    with pytest.raises(RuntimeError, match="2\\^31"):
        tri_mesh(F=Fc).upsample(rounds, True)


# ------------------------------------------------------------------------------------------------ C ABI
def _size(V, F):
    a = lambda n: (n + 255) // 256 * 256
    tiles = (max(V + 1, 3 * F) + 2047) // 2048 + 1
    return a(256) + a(8 * (V + 1)) + a(4 * V) + a(12 * F) + a(24 * F) + a(8 * tiles) + a(12 * F) + a(8 * (3 * F + 1))


def test_abi_declares_and_exports_the_entry_points():
    assert set(ENTRY_POINTS) <= set(_lib.declared_symbols())
    ret, args = _lib.PROTOS["psdf_mesh_subdivide_emit"]
    assert ret == "int" and [a for a, _ in args] == ["V", "F", "smooth", "verts", "faces", "workspace", "verts_out", "faces_out", "stream"]
    assert _lib.PROTOS["psdf_mesh_subdivide_workspace_bytes"][0] == "long long"
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python __graft_entry__.py"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in ENTRY_POINTS:
        assert hasattr(lib, s), "library does not export " + s


@pytest.mark.parametrize("V,F", [(0, 0), (5, 7), (1000, 1999), (2 ** 31 - 1, 2 ** 29 - 1), (3, 2 ** 28)])
def test_workspace_sizes(V, F):
    assert _lib.load_library().psdf_mesh_subdivide_workspace_bytes(V, F) == _size(V, F)


def test_workspace_limits_and_argument_errors():
    lib = _lib.load_library()
    ws = lib.psdf_mesh_subdivide_workspace_bytes
    assert ws(2 ** 31, 1) == -3 and ws(1, 2 ** 29) == -3
    assert ws(-1, 0) == -1 and ws(0, -1) == -1
    assert lib.psdf_mesh_subdivide_count(-1, 0, None, 8, None) == -1
    assert lib.psdf_mesh_subdivide_count(3, 1, None, 8, None) == -1                # faces missing
    assert lib.psdf_mesh_subdivide_count(3, 2 ** 29, 8, 8, None) == -1            # 4F would not fit int32 rows
    assert lib.psdf_mesh_subdivide_emit(3, 1, 1, 8, 8, None, 8, 8, None) == -1    # workspace missing
    assert lib.psdf_mesh_subdivide_emit(3, 1, 0, 8, 8, 8, 8, None, None) == -1    # faces_out missing


# ------------------------------------------------------------------------------------------------ compile check
@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import wgmma_report
    return {r["kernel"]: r for r in wgmma_report.report(("mesh_subdivide.cu",))}


def test_kernels_are_built_and_do_not_spill(kernels):
    sd = {k: r for k, r in kernels.items() if k.startswith(("k_sd_", "k_mesh_"))}
    assert set(sd) == set(KERNELS)
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in sd.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling


# ------------------------------------------------------------------------------------------------ the oracle
@pytest.fixture(scope="module")
def small_meshes():
    V, F = MC.marching_cubes(C.sphere_volume((22,) * 3, (10.3, 10.6, 10.1), 8.0), 0.0)
    keep = V[:, 0] < 10.0
    new_id = np.cumsum(keep) - 1
    return {"sphere": (V, F),
            "torus": MC.marching_cubes(C.torus_volume((30, 30, 14), (14.4, 14.7, 6.6), 9.0, 4.0), 0.0),
            "random": MC.marching_cubes(C.random_field((24, 24, 24), seed=3), 0.0),
            "open": (V[keep], new_id[F[keep[F].all(1)]])}


def nr_edges(F):
    return np.unique(np.sort(C.directed_edges(F), 1), axis=0).shape[0]


@pytest.mark.parametrize("smooth", [False, True])
@pytest.mark.parametrize("name", ["sphere", "torus", "random", "open"])
def test_oracle_counts_and_topology(small_meshes, name, smooth):
    V, F = small_meshes[name]
    Vn, Fn = S.upsample(V, F, 1, smooth)
    assert Vn.shape == (len(V) + nr_edges(F), 3) and Fn.shape == (4 * len(F), 3) and Fn.dtype == np.int32
    assert C.euler_characteristic(Fn) == C.euler_characteristic(F)
    assert C.closed_and_oriented(Fn, len(Vn)) == C.closed_and_oriented(F, len(V))
    if name != "open":
        assert C.closed_and_oriented(Fn, len(Vn))
    if not smooth:
        assert np.array_equal(Vn[:len(V)], V)
    # every edge vertex is the fp32 midpoint (midpoint mode) or lies between its edge's ends; new vertices are numbered by edge
    own, count, _, pos, E = S.edges(np.asarray(F, np.int64), len(V))
    oc = np.nonzero(own == np.arange(own.size))[0]
    u, v = F[oc // 3, oc % 3], F[oc // 3, (oc % 3 + 1) % 3]
    assert np.array_equal(pos[oc], np.arange(E))
    mid = np.float32(0.5) * (V[u] + V[v])
    if not smooth:
        assert np.array_equal(Vn[len(V):], mid)
    else:
        crease = count[oc] != 2
        assert np.array_equal(Vn[len(V):][crease], mid[crease])


def test_tetrahedron_by_hand():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    F = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    # edges in order of their smallest corner: (0,2) (2,1) (1,0) | (1,3) (3,0) | (3,2)
    mids = [(0, 2), (2, 1), (1, 0), (1, 3), (3, 0), (3, 2)]
    Vm, Fm = S.upsample(V, F, 1, False)
    assert np.array_equal(Vm, np.concatenate([V, [(V[a] + V[b]) / 2 for a, b in mids]]))
    assert Fm[:4].tolist() == [[0, 4, 6], [4, 2, 5], [6, 5, 1], [4, 5, 6]]
    Vl, Fl = S.upsample(V, F, 1, True)
    assert np.array_equal(Fl, Fm)
    # n = 3 everywhere: beta = 3/16, p' = 7/16 p + 3/16 (sum of the other three); edge: 3/8 (pu + pv) + 1/8 (the two others)
    even = [7 / 16 * V[i] + 3 / 16 * (V.sum(0) - V[i]) for i in range(4)]
    odd = [3 / 8 * (V[a] + V[b]) + 1 / 8 * (V.sum(0) - V[a] - V[b]) for a, b in mids]
    assert np.array_equal(Vl, np.array(even + odd, np.float32))


def grid_mesh(n):
    x, y = np.meshgrid(np.arange(n + 1, dtype=np.float32), np.arange(n + 1, dtype=np.float32), indexing="ij")
    V = np.stack([x.ravel() * 0.37, y.ravel() * 0.59, np.full(x.size, 2.5, np.float32)], 1).astype(np.float32)
    i = np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]
    i = i.ravel()
    F = np.concatenate([np.stack([i, i + n + 1, i + 1], 1), np.stack([i + 1, i + n + 1, i + n + 2], 1)])
    return V, F


def test_flat_open_grid_stays_flat_and_its_boundary_is_a_crease():
    V, F = grid_mesh(6)
    Vl, Fl = S.upsample(V, F, 2, True)
    assert (Vl[:, 2] == np.float32(2.5)).all()
    assert C.euler_characteristic(Fl) == 1
    # one round: boundary vertices, corners included, have two crease edges and move by the crease rule along the boundary
    V1, _ = S.upsample(V, F, 1, True)
    n = 6
    crease = lambda v, a, b: np.float32(0.75) * V[v] + np.float32(0.125) * (V[a] + V[b])
    b = 3                                             # (0, 3): crease neighbours (0, 2) and (0, 4)
    assert np.array_equal(V1[b], crease(b, b - 1, b + 1)) and V1[b, 0] == V[b, 0]
    assert np.array_equal(V1[0], crease(0, 1, n + 1))
    # an interior vertex has 6 neighbours, all across interior edges
    i = 2 * (n + 1) + 3
    nb = sorted({int(w) for f in F if i in f for w in f if w != i})
    beta = np.float32(3.0) / np.float32(48)
    s = np.zeros(3, np.float32)
    for w in nb:
        s = s + V[w]
    assert len(nb) == 6 and np.array_equal(V1[i], (np.float32(1) - np.float32(6) * beta) * V[i] + beta * s)


def test_non_manifold_fan_keeps_the_edge_vertices():
    V = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0.2], [0.5, 0.1, 1]], np.float32)
    F = np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]])
    Vl, Fl = S.upsample(V, F, 1, True)
    # the edge (0, 1) is in three faces: a crease, so its ends (with k = 4 crease edges each) stay and its vertex is the midpoint
    assert np.array_equal(Vl[:2], V[:2])
    assert np.array_equal(Vl[5], np.float32(0.5) * (V[0] + V[1]))
    # each apex has two crease edges (to 0 and 1) and follows the crease rule
    for a in (2, 3, 4):
        assert np.array_equal(Vl[a], np.float32(0.75) * V[a] + np.float32(0.125) * (V[0] + V[1]))
    assert Fl.shape == (12, 3) and Vl.shape == (5 + 7, 3)
