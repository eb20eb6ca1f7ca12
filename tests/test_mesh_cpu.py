"""Marching cubes without a GPU: the generated triangle table, meshes of analytic and degenerate volumes from the numpy oracle
(oracle/marching_cubes.py, which the GPU kernels must match bit for bit), the PLY writer, vertex cropping and the input checks."""
import math

import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import marching_cubes as M


# ------------------------------------------------------------------------------------------------ table
@pytest.mark.parametrize("cfg", range(256))
def test_table_uses_exactly_the_crossing_edges(cfg):
    crossing = {e for e, (lo, hi) in enumerate(M.EDGE_CORNERS) if (cfg >> lo & 1) != (cfg >> hi & 1)}
    used = {e for tri in M.TABLE[cfg] for e in tri}
    assert used == crossing
    assert all(len(set(tri)) == 3 for tri in M.TABLE[cfg])


@pytest.mark.parametrize("cfg", range(256))
def test_table_interior_edges_twice_once_each_way(cfg):
    """mesh edges inside the cell are used twice, once in each direction; an edge along a cube face is a face segment, used once (the
    cell across the face uses it the other way); no directed edge repeats"""
    directed = [(t[k], t[(k + 1) % 3]) for t in M.TABLE[cfg] for k in range(3)]
    assert len(directed) == len(set(directed))
    segments = {frozenset(s[:2]) for s in M._segments(cfg)}
    for a, b in directed:
        if frozenset((a, b)) in segments:
            assert (b, a) not in directed
        else:
            assert (b, a) in directed
    assert {frozenset(d) for d in directed} >= segments


def test_table_orientation_single_corner():
    """corner 0 inside: one triangle around it with its normal along +(1, 1, 1), away from the inside corner"""
    (tri,) = M.TABLE[1]
    p = [M._mid2(e) / 2.0 for e in tri]
    n = np.cross(p[1] - p[0], p[2] - p[0])
    assert (n > 0).all()


# ------------------------------------------------------------------------------------------------ analytic volumes
CASES = {
    "sphere": lambda: (C.sphere_volume((72, 80, 64), (35.3, 40.1, 31.7), 25.0), 4 / 3 * math.pi * 25 ** 3, 2),
    "torus": lambda: (C.torus_volume((64, 66, 24), (31.6, 32.2, 11.4), 20.0, 7.0), 2 * math.pi ** 2 * 20 * 7 ** 2, 0),
    "touching_spheres": lambda: (C.two_spheres_volume((90, 60, 60), (29.5, 30.2, 29.8), (59.5, 30.2, 29.8), 15.0),
                                 2 * 4 / 3 * math.pi * 15 ** 3, None),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_analytic_volume_mesh(name):
    vol, exact, chi = CASES[name]()
    V, F = M.marching_cubes(vol, 0.0)
    assert V.dtype == np.float32 and F.dtype == np.int32 and F.min() >= 0 and F.max() < len(V)
    assert np.unique(F).size == len(V)
    assert C.closed_and_oriented(F, len(V))
    if chi is not None:
        assert C.euler_characteristic(F) == chi
    vs = C.signed_volume(V, F)
    assert 0 < vs and abs(vs / exact - 1) < 0.02, (vs, exact)
    # vertices on the surface up to the error of linear interpolation along one cell edge (a distance field: O(h^2 / radius))
    if name == "sphere":
        err = np.abs(np.linalg.norm(V - np.array([35.3, 40.1, 31.7]), axis=1) - 25.0)
    elif name == "torus":
        q = np.hypot(V[:, 0] - 31.6, V[:, 1] - 32.2) - 20.0
        err = np.abs(np.hypot(q, V[:, 2] - 11.4) - 7.0)
    else:
        err = np.minimum(np.abs(np.linalg.norm(V - np.array([29.5, 30.2, 29.8]), axis=1) - 15.0),
                         np.abs(np.linalg.norm(V - np.array([59.5, 30.2, 29.8]), axis=1) - 15.0))
    assert err.max() < 0.02, err.max()


def test_random_field_mesh_is_index_closed():
    vol = C.random_field((80, 70, 90), seed=1)
    V, F = M.marching_cubes(vol, 0.0)
    assert len(F) > 1000 and C.balanced(F, len(V)) and C.signed_volume(V, F) > 0


def test_nonzero_threshold_is_the_level_set():
    vol = C.sphere_volume((40, 33, 47), (19.2, 16.1, 23.3), 9.0)
    V, _ = M.marching_cubes(vol, 4.5)
    r = np.linalg.norm(V - np.array([19.2, 16.1, 23.3]), axis=1)
    assert np.abs(r - 13.5).max() < 0.02


# ------------------------------------------------------------------------------------------------ degenerate volumes
def test_exact_threshold_corners_index_closed():
    """values in {-1, 0, 1}: a third of the corners sit exactly on the threshold (outside)"""
    vol = C.pad_outside(np.random.default_rng(0).integers(-1, 2, (20, 17, 23)).astype(np.float32))
    V, F = M.marching_cubes(vol, 0.0)
    assert len(F) > 0 and C.balanced(F, len(V))
    assert all(len(set(f)) == 3 for f in F.tolist())


def test_checkerboard_index_closed():
    """every cell face ambiguous"""
    i, j, k = np.indices((12, 13, 11))
    vol = C.pad_outside(((i + j + k) % 2 * 2 - 1).astype(np.float32))
    V, F = M.marching_cubes(vol, 0.0)
    assert len(F) > 0 and C.balanced(F, len(V))


def test_no_crossing_gives_empty_mesh():
    V, F = M.marching_cubes(np.ones((3, 4, 5), np.float32), 0.0)
    assert V.shape == (0, 3) and F.shape == (0, 3)


# ------------------------------------------------------------------------------------------------ Mesh: PLY and cropping
def test_ply_round_trip(tmp_path):
    from permuto_sdf_b200.mesh import Mesh
    V, F = M.marching_cubes(C.sphere_volume((12, 14, 13), (5.5, 6.2, 6.1), 4.0), 0.0)
    NV = np.random.default_rng(1).standard_normal(V.shape).astype(np.float32)
    m = Mesh(torch.from_numpy(V), torch.from_numpy(F), torch.from_numpy(NV))
    path = tmp_path / "m.ply"
    m.save_to_file(str(path))
    V2, N2, F2 = C.read_ply(str(path))
    assert np.array_equal(V2, V) and np.array_equal(N2, NV) and np.array_equal(F2, F)


def test_remove_marked_vertices():
    from permuto_sdf_b200.mesh import Mesh
    V = torch.arange(15, dtype=torch.float32).view(5, 3)
    NV = -V
    F = torch.tensor([[0, 1, 2], [1, 3, 4], [2, 3, 4], [0, 2, 4]], dtype=torch.int32)
    mask = np.array([True, False, True, True, True])
    kept = Mesh(V.clone(), F.clone(), NV.clone()).remove_marked_vertices(mask, True)
    assert torch.equal(kept.V, V[[0, 2, 3, 4]]) and torch.equal(kept.NV, NV[[0, 2, 3, 4]])
    assert kept.F.dtype == torch.int32 and kept.F.tolist() == [[1, 2, 3], [0, 1, 3]]
    removed = Mesh(V.clone(), F.clone(), NV.clone()).remove_marked_vertices(torch.tensor(mask).view(5, 1), False)
    assert torch.equal(removed.V, V[[1]]) and removed.F.shape == (0, 3)
    with pytest.raises(RuntimeError, match="mask"):
        Mesh(V.clone(), F.clone()).remove_marked_vertices(mask[:4], True)


# ------------------------------------------------------------------------------------------------ refusals
def test_marching_cubes_checks_its_input():
    from permuto_sdf_b200 import marching_cubes
    with pytest.raises(RuntimeError, match="CUDA"):
        marching_cubes(torch.zeros(4, 4, 4))
    with pytest.raises(RuntimeError, match="float32"):
        marching_cubes(torch.zeros(4, 4, 4, dtype=torch.float64))


def test_extract_refuses_a_space_time_sdf():
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    from permuto_sdf_b200.models import SDF
    from permuto_sdf_b200.permuto_sdf import AABB
    m = SDF(4, AABB([1.0, 1.0, 1.0], [0.0, 0.0, 0.0]), 0, 100, nr_levels=8, capacity=2 ** 10)
    with pytest.raises(RuntimeError, match="in_channels 4"):
        extract_mesh_from_sdf_model(m, 16, -0.5, 0.5)
