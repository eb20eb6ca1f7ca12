"""Quadric decimation and vertex normals on the GPU (csrc/mesh_decimate.cu, Mesh.decimate / Mesh.recalculate_normals): V, F, NV and the
round count bit-equal to oracle/decimate.py on marching-cubes meshes at five targets; topology, face counts and non-degenerate faces on
meshes up to 256^3; distance to the analytic surface, face orientation and enclosed volume of decimated spheres and tori; boundaries and
non-manifold edges kept; run-to-run identity, the no-op target and NV = None; and the chained call on a mesh extracted from a fitted
sphere."""
import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import decimate as D
from oracle import marching_cubes as MC

pytestmark = pytest.mark.gpu

TARGETS = (0.9, 0.5, 0.1, 0.01, 0.0)
SPHERE_C, TORUS_C = (21.3, 21.6, 21.1), (25.4, 25.7, 13.6)


def _crop_sphere():
    V, F = MC.marching_cubes(C.sphere_volume((44,) * 3, SPHERE_C, 18.0), 0.0)
    keep = ~((V[:, 0] > 30.0) & (V[:, 2] > 24.0))
    return _remove(V, F, keep)


def _remove(V, F, keep):
    new_id = np.cumsum(keep) - 1
    F = F[keep[F].all(1)]
    return V[keep], new_id[F].astype(np.int32)


def _exact_threshold():
    """integer-valued volume at threshold 0: corners exactly at the threshold give zero-area faces"""
    x, y, z = C.grid((20, 20, 20))
    vol = np.round(np.sqrt((x - 9.5) ** 2 + (y - 9.2) ** 2 + (z - 9.7) ** 2) - 7.0).astype(np.float32)
    return MC.marching_cubes(vol, 0.0)


def bipyramid(n):
    """a ring of n vertices joined to two apexes: closed, the apexes in n faces each (more than the 64 a candidate's end may have)"""
    t = 2 * np.pi * np.arange(n) / n
    V = np.concatenate([np.stack([np.cos(t), np.sin(t), 0.1 * np.sin(3 * t)], 1), [[0, 0, 1.0], [0, 0, -1.0]]]).astype(np.float32)
    i = np.arange(n)
    j = (i + 1) % n
    F = np.concatenate([np.stack([np.full(n, n), i, j], 1), np.stack([np.full(n, n + 1), j, i], 1)]).astype(np.int32)
    return V, F


MESHES = {
    "sphere": lambda: MC.marching_cubes(C.sphere_volume((44,) * 3, SPHERE_C, 18.0), 0.0),
    "torus": lambda: MC.marching_cubes(C.torus_volume((52, 52, 28), TORUS_C, 16.0, 7.0), 0.0),
    "two_spheres": lambda: MC.marching_cubes(C.two_spheres_volume((40, 40, 24), (11.2, 12.3, 11.6), (27.4, 26.1, 11.9), 9.0), 0.0),
    "random": lambda: MC.marching_cubes(C.random_field((40, 40, 40), seed=7), 0.0),
    "exact_threshold": _exact_threshold,
    "cropped_sphere": _crop_sphere,
    "bipyramid": lambda: bipyramid(200),
}
_CACHE = {}


def host_mesh(name):
    if name not in _CACHE:
        V, F = MESHES[name]()
        _CACHE[name] = (np.asarray(V, np.float32), np.asarray(F, np.int32))
    return _CACHE[name]


def gpu_mesh(V, F, normals=True):
    from permuto_sdf_b200.mesh import Mesh
    V = torch.from_numpy(np.ascontiguousarray(V, np.float32)).cuda()
    F = torch.from_numpy(np.ascontiguousarray(F, np.int32)).cuda()
    NV = torch.randn(V.shape, generator=torch.Generator().manual_seed(3)).cuda() if normals else None
    return Mesh(V, F, NV)


def bits(t):
    return t.cpu().numpy().view(np.int32)


# ------------------------------------------------------------------------------------------------ bit for bit against the oracle
@pytest.mark.parametrize("frac", TARGETS)
@pytest.mark.parametrize("name", sorted(MESHES))
def test_decimation_matches_oracle(cuda, name, frac):
    V, F = host_mesh(name)
    target = int(frac * len(F))
    m = gpu_mesh(V, F)
    rounds = m._decimate(target)[3]
    m.decimate(target)
    Vo, Fo, NVo, ro = D.decimate_mesh(V, F, target, True)
    print("%s: %d faces -> %d (target %d) in %d rounds" % (name, len(F), len(Fo), target, ro))
    assert rounds == ro
    assert np.array_equal(bits(m.V), Vo.view(np.int32))
    assert np.array_equal(m.F.cpu().numpy(), Fo)
    assert np.array_equal(bits(m.NV), NVo.view(np.int32))
    if name not in ("exact_threshold", "cropped_sphere") and frac > 0:
        assert len(Fo) in (target, target - 1)


@pytest.mark.parametrize("name", sorted(MESHES))
def test_normals_match_oracle(cuda, name):
    V, F = host_mesh(name)
    m = gpu_mesh(V, F).recalculate_normals()
    assert np.array_equal(bits(m.NV), D.normals(V, F).view(np.int32))


def test_normals_of_vertices_without_faces_are_zero(cuda):
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5]], np.float32)
    m = gpu_mesh(V, np.array([[0, 1, 2]], np.int32)).recalculate_normals()
    assert np.array_equal(m.NV.cpu().numpy(), [[0, 0, 1], [0, 0, 1], [0, 0, 1], [0, 0, 0]])


# ------------------------------------------------------------------------------------------------ topology at scale
def _scale_volumes():
    return [("sphere256", C.sphere_volume((256,) * 3, (127.3, 128.6, 126.9), 110.0)),
            ("torus256", C.torus_volume((256, 256, 128), (127.4, 128.7, 63.6), 80.0, 35.0)),
            ("random128", C.random_field((128, 128, 128), seed=11, sigma=2.5)),
            ("random256", C.random_field((256, 256, 256), seed=12, sigma=2.0))]


def _areas(V, F):
    p = V.astype(np.float64)[F]
    return np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1)


@pytest.mark.parametrize("idx", range(4))
def test_topology_and_faces_at_scale(cuda, idx):
    from permuto_sdf_b200 import marching_cubes
    name, vol = _scale_volumes()[idx]
    V, F = marching_cubes(torch.from_numpy(vol).cuda())
    Fh = F.cpu().numpy()
    # marching cubes of a random field can join four faces at an edge (two blobs touching); decimation keeps such edges as they are
    closed = C.closed_and_oriented(Fh, V.shape[0])
    assert closed or name.startswith("random")
    chi = C.euler_characteristic(Fh)
    # fp32 rounding gives a random field's mesh a few zero-area faces; a collapse never makes another one
    zero_area = int((_areas(V.cpu().numpy(), Fh) == 0).sum())
    assert zero_area == 0 or name.startswith("random")
    ncc = gpu_mesh(V.cpu().numpy(), Fh).remove_small_components(1).connected_components()[1]
    for frac in (0.1, 0.01):
        target = int(frac * F.shape[0])
        m = gpu_mesh(V.cpu().numpy(), Fh)
        m.decimate(target)
        Fd, Vd = m.F.cpu().numpy(), m.V.cpu().numpy()
        print("%s: %d faces -> %d (target %d), %d components" % (name, F.shape[0], len(Fd), target, ncc))
        assert C.closed_and_oriented(Fd, len(Vd)) == closed and C.balanced(Fd, len(Vd))
        assert C.euler_characteristic(Fd) == chi
        assert m.connected_components()[1] == ncc
        assert (_areas(Vd, Fd) == 0).sum() <= zero_area
        if frac == 0.1:
            assert len(Fd) in (target, target - 1)


# ------------------------------------------------------------------------------------------------ geometry on analytic surfaces
# bars set from oracle/decimate.py on these meshes (measured: sphere 0.27 % / 2.4 % of the radius, volume 0.19 % / 2.2 %; torus 0.80 % /
# 8.4 % of the tube radius, volume 0.28 % / 3.6 %, at 10 % / 1 % of the faces)
GEOMETRY = {("sphere", 0.1): (0.006, 0.005), ("sphere", 0.01): (0.04, 0.035),
            ("torus", 0.1): (0.015, 0.005), ("torus", 0.01): (0.12, 0.05)}


@pytest.mark.parametrize("name,frac", sorted(GEOMETRY))
def test_geometry_on_analytic_surfaces(cuda, name, frac):
    if name == "sphere":
        c, vol = np.array((27.3, 27.6, 27.1)), C.sphere_volume((56,) * 3, (27.3, 27.6, 27.1), 24.0)
    else:
        c, vol = np.array((31.4, 31.7, 15.6)), C.torus_volume((64, 64, 32), (31.4, 31.7, 15.6), 20.0, 9.0)
    V, F = MC.marching_cubes(vol, 0.0)
    m = gpu_mesh(V, F).decimate(int(frac * len(F)))
    Vd, Fd = m.V.cpu().numpy().astype(np.float64), m.F.cpu().numpy()
    q = Vd - c
    if name == "sphere":
        dist, rad = np.linalg.norm(q, axis=1) - 24.0, 24.0
        normal = lambda x: x
    else:
        dist, rad = np.hypot(np.hypot(q[:, 0], q[:, 1]) - 20.0, q[:, 2]) - 9.0, 9.0

        def normal(x):
            rho = np.hypot(x[:, 0], x[:, 1])
            return x - 20.0 * np.stack([x[:, 0] / rho, x[:, 1] / rho, 0 * rho], 1)
    bar_r, bar_v = GEOMETRY[(name, frac)]
    assert np.abs(dist).max() <= bar_r * rad
    p = Vd[Fd]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert (np.einsum("ij,ij->i", n, normal(p.mean(1) - c)) > 0).all()
    assert abs(C.signed_volume(Vd, Fd) / C.signed_volume(V, F) - 1) <= bar_v


# ------------------------------------------------------------------------------------------------ open and non-manifold input
def _boundary_edges(V, F):
    e = C.directed_edges(F)
    keys = set(map(tuple, e.tolist()))
    return {tuple(sorted((tuple(V[a]), tuple(V[b])))) for a, b in e.tolist() if (b, a) not in keys}


@pytest.mark.parametrize("frac", (0.1, 0.0))
def test_boundary_is_kept(cuda, frac):
    V, F = host_mesh("cropped_sphere")
    before = _boundary_edges(V, F)
    assert before
    m = gpu_mesh(V, F).decimate(int(frac * len(F)))
    assert len(m.F) < len(F) // 5
    assert _boundary_edges(m.V.cpu().numpy(), m.F.cpu().numpy()) == before


def test_edge_of_three_faces_is_kept(cuda):
    V, F = host_mesh("sphere")
    # a fin: a third face on an edge of the sphere, with a vertex of its own
    a, b = int(F[100, 0]), int(F[100, 1])
    V2 = np.concatenate([V, [V[a] + 3.0 * (V[a] - SPHERE_C) / 18.0]]).astype(np.float32)
    F2 = np.concatenate([F, [[a, b, len(V)]]]).astype(np.int32)
    m = gpu_mesh(V2, F2)
    Vd, Fd, removed, _ = m._decimate(int(0.05 * len(F2)))
    assert not removed[[a, b, len(V)]].any().item()
    assert np.array_equal(bits(Vd[[a, b, len(V)]]), V2[[a, b, len(V)]].view(np.int32))
    assert len(Fd) < len(F2) // 10


def test_vertices_of_high_valence(cuda):
    """two apexes in 10^5 faces each: the per-vertex work stays bounded (heap sort, twins looked up at the end with fewer faces, no
    candidate with an end in more than 64 faces), and the apexes stay while they are in more than 64 faces"""
    import time
    n = 100000
    V, F = bipyramid(n)
    m = gpu_mesh(V, F)
    torch.cuda.synchronize()
    t = time.perf_counter()
    m.decimate(1000)
    torch.cuda.synchronize()
    print("bipyramid of %d faces -> %d in %.3f s" % (len(F), len(m.F), time.perf_counter() - t))
    Vd, Fd = m.V.cpu().numpy(), m.F.cpu().numpy()
    assert len(Fd) in (1000, 999)
    assert C.closed_and_oriented(Fd, len(Vd)) and C.euler_characteristic(Fd) == 2
    assert np.array_equal(bits(m.V[-2:]), V[-2:].view(np.int32))
    assert (np.bincount(Fd.reshape(-1), minlength=len(Vd))[-2:] == 500).all()


# ------------------------------------------------------------------------------------------------ contract
def test_same_bits_on_every_call(cuda):
    V, F = host_mesh("random")
    a = gpu_mesh(V, F).decimate(len(F) // 20)
    b = gpu_mesh(V, F).decimate(len(F) // 20)
    assert torch.equal(a.V, b.V) and torch.equal(a.F, b.F) and torch.equal(a.NV, b.NV)


@pytest.mark.parametrize("extra", (0, 1, 1000))
def test_target_at_or_above_the_face_count_is_a_no_op(cuda, extra):
    V, F = host_mesh("torus")
    m = gpu_mesh(V, F)
    V0, F0, N0 = m.V.clone(), m.F.clone(), m.NV.clone()
    assert m.decimate(len(F) + extra) is m
    assert torch.equal(m.V, V0) and torch.equal(m.F, F0) and torch.equal(m.NV, N0)


def test_absent_normals_stay_absent(cuda):
    V, F = host_mesh("sphere")
    m = gpu_mesh(V, F, normals=False).decimate(len(F) // 10)
    assert m.NV is None and len(m.F) in (len(F) // 10, len(F) // 10 - 1)


def test_unreferenced_vertices_are_kept(cuda):
    V, F = host_mesh("sphere")
    V2 = np.concatenate([V, [[100.0, 100.0, 100.0]]]).astype(np.float32)
    m = gpu_mesh(V2, F).decimate(len(F) // 10)
    assert m.V[-1].tolist() == [100.0, 100.0, 100.0] and m.NV[-1].tolist() == [0.0, 0.0, 0.0]


def test_bad_faces_are_refused(cuda):
    V, F = host_mesh("sphere")
    for bad, match in ((len(V), "outside"), (-1, "outside")):
        F2 = F.copy()
        F2[7, 1] = bad
        with pytest.raises(RuntimeError, match=match):
            gpu_mesh(V, F2).decimate(10)
        with pytest.raises(RuntimeError, match=match):
            gpu_mesh(V, F2).recalculate_normals()
    F2 = F.copy()
    F2[7, 1] = F2[7, 2]
    with pytest.raises(RuntimeError, match="repeat"):
        gpu_mesh(V, F2).decimate(10)
    with pytest.raises(RuntimeError, match="repeat"):
        gpu_mesh(V, F2).recalculate_normals()
    V2 = V.copy()
    V2[3, 0] = np.nan
    with pytest.raises(RuntimeError, match="finite"):
        gpu_mesh(V2, F).decimate(10)


def test_chained_on_a_fitted_sphere(cuda):
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    from permuto_sdf_b200.train import HyperParams, Trainer
    tr = Trainer(HyperParams(), nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=128, nr_images=4, seed=5,
                 optimizer="fused")
    tr.set_analytic_scene()
    tr.fit_sphere()
    mesh = extract_mesh_from_sdf_model(tr.model_sdf, 256, -0.5, 0.5).keep_largest_component()
    nf = len(mesh.F)
    mesh.decimate(nf // 50)
    Fd, Vd = mesh.F.cpu().numpy(), mesh.V.cpu().numpy()
    print("fitted sphere: %d faces -> %d" % (nf, len(Fd)))
    assert len(Fd) in (nf // 50, nf // 50 - 1)
    assert C.closed_and_oriented(Fd, len(Vd)) and C.euler_characteristic(Fd) == 2
    assert np.abs(np.linalg.norm(Vd, axis=1) - 0.3).max() < 0.03
    assert mesh.NV is not None and np.allclose(np.linalg.norm(mesh.NV.cpu().numpy(), axis=1), 1, atol=1e-5)
