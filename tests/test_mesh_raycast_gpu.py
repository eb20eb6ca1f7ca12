"""Mesh.occluded and Mesh.ambient_occlusion on the GPU against the brute-force oracle (oracle/raycast.py), bit for bit, on triangle soups,
marching-cubes meshes, axis-aligned meshes with zero-thickness boxes, degenerate and duplicate faces, and rays aimed at edges, vertices and
box planes; the known answers of ambient occlusion; Mesh.interpolate."""
import math

import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import raycast as RC
from permuto_sdf_b200.mesh import Mesh, marching_cubes

pytestmark = pytest.mark.gpu


def cu(a, dt=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)


def check(V, F, o, d, tnear=1e-4, tfar=math.inf, expect_some=True):
    m = Mesh(cu(V), cu(np.asarray(F).reshape(-1, 3), torch.int32))
    got = m.occluded(cu(o), cu(d), tnear, tfar).cpu().numpy()
    ref = RC.occluded(V, F, o, d, np.float32(tnear), tfar)
    bad = np.flatnonzero(got != ref)
    assert bad.size == 0, (bad.size, bad[:10], o[bad[:3]], d[bad[:3]])
    if expect_some:
        assert 0 < ref.sum() < ref.size
    return ref


def rand_dirs(rng, n):
    d = rng.standard_normal((n, 3))
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def mc_mesh(vol):
    V, F = marching_cubes(cu(vol))
    return V.cpu().numpy(), F.cpu().numpy()


def box_mesh(lo, hi):
    x = np.array([[lo[0], lo[1], lo[2]], [hi[0], lo[1], lo[2]], [hi[0], hi[1], lo[2]], [lo[0], hi[1], lo[2]],
                  [lo[0], lo[1], hi[2]], [hi[0], lo[1], hi[2]], [hi[0], hi[1], hi[2]], [lo[0], hi[1], hi[2]]], np.float32)
    F = np.array([[0, 2, 1], [0, 3, 2], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4], [2, 3, 7], [2, 7, 6], [1, 2, 6], [1, 6, 5],
                  [0, 4, 7], [0, 7, 3]])
    return x, F


def floor_grid(n, h=0.25, z=0.0):
    x, y = np.meshgrid(np.arange(n + 1) * h, np.arange(n + 1) * h, indexing="ij")
    V = np.stack([x.ravel(), y.ravel(), np.full(x.size, z)], 1).astype(np.float32)
    i = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]).ravel()
    return V, np.concatenate([np.stack([i, i + n + 1, i + 1], 1), np.stack([i + 1, i + n + 1, i + n + 2], 1)])


# ------------------------------------------------------------------------------------------------ occluded == brute force
@pytest.mark.parametrize("seed", [0, 1])
def test_random_soups(cuda, seed):
    rng = np.random.default_rng(seed)
    F = 1500
    c = rng.uniform(-1, 1, (F, 1, 3))
    V = (c + rng.standard_normal((F, 3, 3)) * rng.uniform(0.001, 0.2, (F, 1, 1))).reshape(-1, 3).astype(np.float32)
    o = rng.uniform(-1.5, 1.5, (20000, 3)).astype(np.float32)
    check(V, np.arange(3 * F).reshape(-1, 3), o, rand_dirs(rng, 20000))
    check(V, np.arange(3 * F).reshape(-1, 3), o, rand_dirs(rng, 20000) * np.float32(7.5), tnear=0.0, tfar=0.3)


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_marching_cubes_meshes(cuda, name):
    vol = C.sphere_volume((30,) * 3, (14.3, 14.6, 14.1), 11.0) if name == "sphere" else C.torus_volume((40, 40, 20), (19.4, 19.7, 9.6),
                                                                                                          13.0, 5.0)
    V, F = mc_mesh(vol)
    rng = np.random.default_rng(3)
    lo, hi = V.min(0) - 2, V.max(0) + 2
    o = rng.uniform(lo, hi, (8000, 3)).astype(np.float32)
    check(V, F, o, rand_dirs(rng, 8000))
    # from the vertices themselves, as ambient occlusion casts them
    idx = rng.integers(0, V.shape[0], 8000)
    check(V, F, V[idx], rand_dirs(rng, 8000))


def test_axis_aligned_box_and_floor(cuda):
    """zero-thickness boxes; axis-parallel rays, origins on box planes, rays aimed at shared edges and vertices, grazing rays"""
    bV, bF = box_mesh((0.0, 0.0, 0.0), (1.0, 2.0, 0.5))
    gV, gF = floor_grid(8, z=-1.0)
    V = np.concatenate([bV, gV])
    F = np.concatenate([bF, gF + bV.shape[0]])
    rng = np.random.default_rng(5)
    axes = np.concatenate([np.eye(3), -np.eye(3)]).astype(np.float32)
    grid = np.arange(-2, 10) * np.float32(0.25)
    # origins on the planes of the box and the floor, at edge and vertex coordinates, and in between
    pts = np.stack(np.meshgrid(grid, grid, np.array([-1.0, -0.5, 0.0, 0.25, 0.5, 1.0], np.float32), indexing="ij"), -1).reshape(-1, 3)
    o = np.repeat(pts, 6, 0).astype(np.float32)
    d = np.tile(axes, (pts.shape[0], 1))
    check(V, F, o, d, tnear=-1e-4)
    check(V, F, o, d, tnear=1e-4)
    # aimed exactly at grid vertices and edge midpoints of the floor from above, and at box corners and edges
    tgt = np.concatenate([gV, (gV[gF[:, 0]] + gV[gF[:, 1]]) / 2, bV, (bV[bF[:, 0]] + bV[bF[:, 2]]) / 2]).astype(np.float32)
    src = (tgt + rng.uniform(-3, 3, tgt.shape)).astype(np.float32)
    check(V, F, src, (tgt - src).astype(np.float32), tnear=0.0)
    # grazing: nearly in the floor's plane and in the box's faces, and exactly in them
    n = 6000
    o = np.concatenate([rng.uniform(-0.5, 2.5, (n, 2)), np.full((n, 1), -1.0) + rng.choice([0.0, 1e-6, -1e-6], (n, 1))], 1).astype(np.float32)
    d = np.concatenate([rand_dirs(rng, n)[:, :2], rng.choice([0.0, 1e-3, -1e-3, 1e-7], (n, 1))], 1).astype(np.float32)
    check(V, F, o, d, tnear=-1.0)
    o2 = np.concatenate([rng.uniform(-0.5, 1.5, (n, 1)), rng.uniform(-0.5, 2.5, (n, 1)), np.full((n, 1), 0.5)], 1).astype(np.float32)
    check(V, F, o2, d, tnear=-1.0)


def test_duplicates_equal_centroids_and_tiny_meshes(cuda):
    rng = np.random.default_rng(7)
    # 64 triangles rotated about one centroid, each twice, and faces that repeat a vertex
    ang = np.linspace(0, 2 * np.pi, 64, endpoint=False)[:, None] + np.array([0, 2 * np.pi / 3, 4 * np.pi / 3])[None]
    tri = np.stack([np.cos(ang), np.sin(ang), np.zeros_like(ang)], -1) * 0.5
    tri[..., 2] = np.linspace(-0.1, 0.1, 64)[:, None] * np.array([1, -1, 0])[None]
    V = np.concatenate([tri.reshape(-1, 3), tri.reshape(-1, 3)]).astype(np.float32)
    F = np.concatenate([np.arange(V.shape[0]).reshape(-1, 3), [[0, 0, 1], [2, 2, 2]]])
    o = rng.uniform(-1, 1, (20000, 3)).astype(np.float32)
    d = rand_dirs(rng, 20000)
    check(V, F, o, d)
    # all faces at one point: nothing is hit
    check(np.zeros((9, 3), np.float32), np.arange(9).reshape(-1, 3), o, d, expect_some=False)
    # F = 1 and F = 0
    check(V[:3], [[0, 1, 2]], o, d)
    assert not check(V[:3], np.zeros((0, 3), int), o, d, expect_some=False).any()


@pytest.mark.parametrize("R", [1, 255, 256, 257, 2 ** 20 + 3])
def test_ray_counts(cuda, R):
    rng = np.random.default_rng(R)
    V, F = box_mesh((-0.5, -0.25, -0.75), (0.5, 0.75, 0.25))
    o = rng.uniform(-1, 1, (R, 3)).astype(np.float32)
    d = rand_dirs(rng, R)
    check(V, F, o, d, expect_some=R > 1000)


# ------------------------------------------------------------------------------------------------ ambient occlusion
def rotation(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((3, 3)))
    return q


def two_spheres():
    """concentric marching-cubes spheres, rotated: a marching-cubes mesh has rows of vertices and edges in the grid planes, and a ray
    running in such a plane meets them exactly on shared edges, where the fp32 test may pass neither face"""
    outer = C.sphere_volume((40,) * 3, (19.3, 19.6, 19.1), 16.0)
    inner = C.sphere_volume((40,) * 3, (19.3, 19.6, 19.1), 6.0)
    oV, oF = mc_mesh(outer)
    iV, iF = mc_mesh(inner)
    V = (np.concatenate([oV, iV]).astype(np.float64) - 19.3) @ rotation(11).T
    return V.astype(np.float32), np.concatenate([oF, iF + oV.shape[0]]), oV.shape[0]


def test_ambient_occlusion_matches_occluded_and_the_oracle(cuda):
    V, F = mc_mesh(C.torus_volume((36, 36, 18), (17.4, 17.7, 8.6), 11.0, 4.5))
    m = Mesh(cu(V), cu(F, torch.int32)).recalculate_normals()
    S = 37
    vis = m.ambient_occlusion(S)
    assert vis.dtype == torch.float32 and vis.shape == (V.shape[0],)
    o, d = RC.ao_rays(V, m.NV.cpu().numpy(), S)
    hits = m.occluded(cu(o), cu(d)).view(-1, S).sum(1).cpu().numpy()
    from_occluded = ((S - hits).astype(np.float32) / np.float32(S)).astype(np.float32)
    assert np.array_equal(vis.cpu().numpy(), from_occluded)
    assert np.array_equal(vis.cpu().numpy(), RC.ambient_occlusion(V, F, m.NV.cpu().numpy(), S))
    assert 0 < float(vis.min()) < 1 and float(vis.max()) == 1
    assert torch.equal(m.ambient_occlusion(S), vis)


def test_ambient_occlusion_known_answers(cuda):
    V, F, n_outer = two_spheres()
    m = Mesh(cu(V), cu(F, torch.int32)).recalculate_normals()
    vis = m.ambient_occlusion(100)
    assert torch.equal(vis, m.ambient_occlusion(100))
    assert (vis[n_outer:] == 0).all(), "a closed sphere inside a larger closed sphere sees nothing"
    assert float(vis[:n_outer].min()) > 0.5
    # nothing to occlude: exactly 1
    e = Mesh(cu(V), torch.zeros(0, 3, dtype=torch.int32, device="cuda"), m.NV)
    assert (e.ambient_occlusion(100) == 1).all()


def test_ambient_occlusion_in_a_right_angled_corner(cuda):
    """a vertex 1e-3 inside the edge of a 90 degree dihedral of two planes of side 2000 (y = 0 and z = 0), normal along the bisector: of
    the hemisphere around it, exactly the quarter-space y, z > 0 is open, half of the hemisphere"""
    L = 1000.0
    V = np.array([[-L, 0, 0], [L, 0, 0], [L, L, 0], [-L, L, 0], [-L, 0, L], [L, 0, L], [1e-3, 1e-3, 1e-3]], np.float32)
    F = np.array([[0, 1, 2], [0, 2, 3], [0, 4, 5], [0, 5, 1]])
    NV = np.zeros_like(V)
    NV[6] = np.float32([0, 1, 1]) / np.float32(math.sqrt(2))
    m = Mesh(cu(V), cu(F, torch.int32), cu(NV))
    vis = float(m.ambient_occlusion(4096)[6])
    assert abs(vis - 0.5) < 0.02, vis


def test_refusals(cuda):
    V, F = box_mesh((0, 0, 0), (1, 1, 1))
    m = Mesh(cu(V), cu(F, torch.int32))
    with pytest.raises(RuntimeError, match="recalculate_normals"):
        m.ambient_occlusion(100)
    m.recalculate_normals()
    bad = Mesh(m.V, cu(np.concatenate([F, [[0, 1, 8]]]), torch.int32), torch.zeros(8, 3, device="cuda"))
    with pytest.raises(RuntimeError, match="outside"):
        bad.ambient_occlusion(10)
    with pytest.raises(RuntimeError, match="outside"):
        bad.occluded(torch.zeros(1, 3, device="cuda"), torch.ones(1, 3, device="cuda"))
    Vn = m.V.clone()
    Vn[3, 1] = float("nan")
    with pytest.raises(RuntimeError, match="finite"):
        Mesh(Vn, m.F, m.NV).ambient_occlusion(10)
    with pytest.raises(RuntimeError, match="finite"):
        m.occluded(torch.full((1, 3), float("inf"), device="cuda"), torch.ones(1, 3, device="cuda"))
    # faces that repeat a vertex are allowed and never hit
    rep = Mesh(m.V, cu(np.concatenate([F, [[0, 0, 6]]]), torch.int32), m.NV)
    assert torch.equal(rep.ambient_occlusion(16), m.ambient_occlusion(16))


# ------------------------------------------------------------------------------------------------ interpolate
def test_interpolate(cuda):
    V, F = mc_mesh(C.sphere_volume((16,) * 3, (7.3, 7.6, 7.1), 5.0))
    a = Mesh(cu(V), cu(F, torch.int32)).recalculate_normals()
    b = Mesh(a.V * 1.5 + 0.25, a.F.clone())
    for t in (0.0, 0.05, 0.5, 0.95, 1.0):
        r = a.interpolate(b, t)
        assert torch.equal(r.V, torch.lerp(a.V, b.V, t)) and torch.equal(r.F, a.F) and r.NV is None
    with pytest.raises(RuntimeError, match="different faces"):
        a.interpolate(Mesh(b.V, b.F.flip(1)), 0.5)
    with pytest.raises(RuntimeError, match="shape"):
        a.interpolate(Mesh(b.V[1:], b.F), 0.5)
