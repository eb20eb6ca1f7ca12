"""Mesh.closest_points, Mesh.signed_distance and mesh_distance on the GPU: dist2, face and bary against the brute-force oracle
(oracle/mesh_distance.py) bit for bit on triangle soups, rotated marching-cubes meshes, a box over a grid, duplicate and degenerate faces and
points on vertices and edges; the sign against analytic inside / outside; mesh distances against an fp64 oracle and known answers; and a
fitted SDF checked against the true signed distance of its mesh."""
import math

import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import mesh_distance as MD
from permuto_sdf_b200._lib import call
from permuto_sdf_b200.mesh import Mesh, marching_cubes, mesh_distance
from test_mesh_raycast_gpu import box_mesh, cu, floor_grid, mc_mesh, rotation

pytestmark = pytest.mark.gpu


def raw(V, F, P):
    """psdf_mesh_closest_points -> (dist2, face, bary) as numpy"""
    m = Mesh(cu(V), cu(np.asarray(F).reshape(-1, 3), torch.int32))
    _, _, _, d2, face, bary = m._closest("test", cu(P))
    return d2.cpu().numpy(), face.cpu().numpy(), bary.cpu().numpy()


def check(V, F, P):
    d2, face, bary = raw(V, F, P)
    r2, rf, rb = MD.closest_points(V, F, P)
    bad = np.flatnonzero((d2.view(np.uint32) != r2.view(np.uint32)) | (face != rf) | (bary.view(np.uint32) != rb.view(np.uint32)).any(1))
    assert bad.size == 0, (bad.size, bad[:5], P[bad[:3]], d2[bad[:3]], r2[bad[:3]], face[bad[:3]], rf[bad[:3]], bary[bad[:3]], rb[bad[:3]])
    return r2, rf


def near_and_uniform(rng, V, n, spread):
    lo, hi = V.min(0) - spread, V.max(0) + spread
    near = V[rng.integers(0, V.shape[0], n)] + rng.standard_normal((n, 3)) * spread * 0.05
    return np.concatenate([near, rng.uniform(lo, hi, (n, 3))]).astype(np.float32)


def rotated_mc(name):
    if name == "sphere":
        V, F = mc_mesh(C.sphere_volume((30,) * 3, (14.3, 14.6, 14.1), 11.0))
    else:
        V, F = mc_mesh(C.torus_volume((40, 40, 20), (19.4, 19.7, 9.6), 13.0, 5.0))
    c = V.mean(0)
    return ((V.astype(np.float64) - c) @ rotation(11).T).astype(np.float32), F


# ------------------------------------------------------------------------------------------------ closest points == brute force
@pytest.mark.parametrize("seed", [0, 1])
def test_random_soups(cuda, seed):
    rng = np.random.default_rng(seed)
    F = 1500
    c = rng.uniform(-1, 1, (F, 1, 3))
    V = (c + rng.standard_normal((F, 3, 3)) * rng.uniform(0.001, 0.2, (F, 1, 1))).reshape(-1, 3).astype(np.float32)
    check(V, np.arange(3 * F).reshape(-1, 3), rng.uniform(-1.5, 1.5, (4000, 3)).astype(np.float32))


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_rotated_marching_cubes_meshes(cuda, name):
    V, F = rotated_mc(name)
    rng = np.random.default_rng(3)
    P = near_and_uniform(rng, V, 1000, 2.0)
    # on the vertices, on edge midpoints and at face centroids
    e = rng.integers(0, F.shape[0], 500)
    on = np.concatenate([V[rng.integers(0, V.shape[0], 500)], (V[F[e, 0]] + V[F[e, 1]]) / 2, V[F[e]].mean(1)]).astype(np.float32)
    d2, _ = check(V, F, np.concatenate([P, on]))
    assert (d2[-1500:-1000] == 0).all()


def test_box_over_a_grid(cuda):
    """axis-aligned faces; points on the box and floor planes, on their vertices and edges, and on the grid's lines"""
    bV, bF = box_mesh((0.0, 0.0, 0.0), (1.0, 2.0, 0.5))
    gV, gF = floor_grid(8, z=-1.0)
    V = np.concatenate([bV, gV])
    F = np.concatenate([bF, gF + bV.shape[0]])
    g = np.arange(-2, 10) * np.float32(0.25)
    P = np.stack(np.meshgrid(g, g, np.array([-1.5, -1.0, -0.5, 0.0, 0.25, 0.5, 1.0], np.float32), indexing="ij"), -1).reshape(-1, 3)
    mids = np.concatenate([(V[F[:, 0]] + V[F[:, 1]]) / 2, (V[F[:, 1]] + V[F[:, 2]]) / 2, V]).astype(np.float32)
    rng = np.random.default_rng(5)
    check(V, F, np.concatenate([P.astype(np.float32), mids, rng.uniform(-1, 3, (4000, 3)).astype(np.float32)]))


def test_duplicates_degenerate_faces_and_tiny_meshes(cuda):
    rng = np.random.default_rng(7)
    V, F = rotated_mc("sphere")
    # every face twice (ties go to the lower index), once more with its corners rotated, faces that repeat a vertex, and a sliver whose
    # third corner is the fp32-rounded midpoint of an edge (zero-area faces are the all-at-one-point and `line` meshes below)
    col = np.array([[F[0, 0], F[0, 1], V.shape[0]]])
    Vc = np.concatenate([V, [(V[F[0, 0]] + V[F[0, 1]]) / 2]]).astype(np.float32)
    F2 = np.concatenate([F[:300], F[:300], F[:300, [1, 2, 0]], [[0, 0, 1], [2, 2, 2]], col])
    P = np.concatenate([near_and_uniform(rng, V, 1500, 2.0), Vc[-1:], Vc[F[:50, 0]]]).astype(np.float32)
    _, face = check(Vc, F2, P)
    assert (face < 300).any() and not np.isin(face, [900, 901]).any()
    # all faces at one point, and collinear faces alone
    check(np.zeros((9, 3), np.float32), np.arange(9).reshape(-1, 3), P)
    line = np.array([[0, 0, 0], [2, 0, 0], [1, 0, 0], [3, 0, 0]], np.float32)
    check(line, np.array([[0, 1, 2], [1, 3, 2]]), P / 4)
    # F = 1 and F = 0
    check(V[:3], np.array([[0, 1, 2]]), P)
    d2, face, bary = raw(V, np.zeros((0, 3), int), P)
    assert np.isinf(d2).all() and (face == -1).all() and (bary == 0).all()
    m = Mesh(cu(V), cu(np.zeros((0, 3), int), torch.int32))
    dist, face, q = m.closest_points(cu(P[:4]))
    assert torch.isinf(dist).all() and (face == -1).all() and torch.isnan(q).all()
    assert torch.isinf(m.signed_distance(cu(P[:4]))).all()


@pytest.mark.parametrize("P", [1, 255, 256, 257, 2 ** 20 + 3])
def test_point_counts(cuda, P):
    rng = np.random.default_rng(P)
    V, F = box_mesh((-0.5, -0.25, -0.75), (0.5, 0.75, 0.25))
    check(V, F, rng.uniform(-1, 1, (P, 3)).astype(np.float32))


def test_closest_points_returns_the_point(cuda):
    V, F = rotated_mc("torus")
    rng = np.random.default_rng(9)
    P = near_and_uniform(rng, V, 800, 2.0)
    m = Mesh(cu(V), cu(F, torch.int32))
    dist, face, q = m.closest_points(cu(P))
    r2, rf, rb = MD.closest_points(V, F, P)
    assert torch.equal(dist, torch.sqrt(cu(r2))) and np.array_equal(face.cpu().numpy(), rf)
    corners = V[F[rf]]
    rq = (rb[:, 0:1] * corners[:, 0] + rb[:, 1:2] * corners[:, 1]) + rb[:, 2:3] * corners[:, 2]
    assert np.allclose(q.cpu().numpy(), rq, rtol=0, atol=1e-5)
    assert np.allclose(np.linalg.norm(P - q.cpu().numpy(), axis=1), dist.cpu().numpy(), rtol=1e-4, atol=1e-5)


def test_refusals(cuda):
    V, F = box_mesh((0, 0, 0), (1, 1, 1))
    m = Mesh(cu(V), cu(F, torch.int32))
    bad = Mesh(m.V, cu(np.concatenate([F, [[0, 1, 8]]]), torch.int32))
    p = torch.zeros(1, 3, device="cuda")
    for f in (bad.closest_points, bad.signed_distance):
        with pytest.raises(RuntimeError, match="outside"):
            f(p)
    with pytest.raises(RuntimeError, match="finite"):
        m.closest_points(torch.full((1, 3), float("nan"), device="cuda"))
    with pytest.raises(RuntimeError, match=r"\[P,3\]"):
        m.signed_distance(torch.zeros(4, device="cuda"))
    flat = Mesh(cu(np.zeros((3, 3), np.float32)), cu([[0, 1, 2]], torch.int32))
    with pytest.raises(RuntimeError, match="positive area"):
        mesh_distance(flat, m, nr_samples=10)
    for x, y in ((bad, m), (m, bad)):
        with pytest.raises(RuntimeError, match="outside"):
            mesh_distance(x, y, nr_samples=10)


# ------------------------------------------------------------------------------------------------ signed distance
def sphere_sdf(P, r):
    return np.linalg.norm(P.astype(np.float64), axis=1) - r


def torus_sdf(P, R, r):
    P = P.astype(np.float64)
    q = np.linalg.norm(P[:, :2], axis=1) - R
    return np.hypot(q, P[:, 2]) - r


def shapes():
    """closed, outward meshes with their analytic SDF: a rotated marching-cubes sphere and torus, and a box"""
    Q = rotation(4)
    sV, sF = mc_mesh(C.sphere_volume((40,) * 3, (19.3, 19.6, 19.1), 15.0))
    sV = ((sV.astype(np.float64) - [19.3, 19.6, 19.1]) @ Q.T).astype(np.float32)
    tV, tF = mc_mesh(C.torus_volume((48, 48, 24), (23.4, 23.7, 11.6), 15.0, 6.0))
    tV = ((tV.astype(np.float64) - [23.4, 23.7, 11.6]) @ Q.T).astype(np.float32)
    bV, bF = box_mesh((-1.0, -2.0, -0.5), (1.5, 1.0, 0.75))

    def box_sdf(P):
        c, h = np.array([0.25, -0.5, 0.125]), np.array([1.25, 1.5, 0.625])
        q = np.abs(P.astype(np.float64) - c) - h
        return np.linalg.norm(np.maximum(q, 0), axis=1) + np.minimum(q.max(1), 0)
    return [("sphere", sV, sF, lambda P: sphere_sdf(P @ Q, 15.0)), ("torus", tV, tF, lambda P: torus_sdf(P @ Q, 15.0, 6.0)),
            ("box", bV, bF, box_sdf)]


def deviation(m, true_sdf, V):
    """how far the mesh strays from the analytic surface: |true sdf| at the vertices and at 10^5 surface samples"""
    pts, _ = m._sample_surface("test", 100000, 5)
    return max(np.abs(true_sdf(V)).max(), np.abs(true_sdf(pts.cpu().numpy())).max())


@pytest.mark.parametrize("which", [0, 1, 2])
def test_sign_against_analytic_inside_and_outside(cuda, which):
    name, V, F, true_sdf = shapes()[which]
    assert C.closed_and_oriented(F, V.shape[0])
    m = Mesh(cu(V), cu(F, torch.int32))
    rng = np.random.default_rng(which)
    P = near_and_uniform(rng, V, 30000, float(np.ptp(V, 0).max()) * 0.2)
    sdf = m.signed_distance(cu(P))
    dist, face, _ = m.closest_points(cu(P))
    s, d = sdf.cpu().numpy(), dist.cpu().numpy()
    assert np.array_equal(np.abs(s)[s != 0], d[s != 0]) and (s == 0).mean() < 1e-3
    t = true_sdf(P)
    clear = np.abs(t) > deviation(m, true_sdf, V) + 1e-3
    assert clear.sum() > 20000
    wrong = np.flatnonzero(clear & ((s < 0) != (t < 0)))
    assert wrong.size == 0, (name, wrong.size, P[wrong[:5]], s[wrong[:5]], t[wrong[:5]])
    # where the fp64 oracle's cosine of p - q and the pseudonormal exceeds 1e-3, the fp32 sign agrees with it as well
    _, rf, rb = MD.closest_points(V, F, P[:2000])
    cos = MD.signed_cos(V, F, P[:2000], rf, rb)
    big = np.abs(cos) > 1e-3
    assert big.mean() > 0.9 and np.array_equal(np.sign(cos[big]), np.sign(s[:2000][big]))
    assert torch.equal(m.signed_distance(cu(P)), sdf)


def test_fine_sphere_is_within_its_chord_error(cuda):
    r = 60.0
    V, F = mc_mesh(C.sphere_volume((128,) * 3, (63.3, 63.6, 63.1), r))
    V = (V - np.float32([63.3, 63.6, 63.1])).astype(np.float32)
    m = Mesh(cu(V), cu(F, torch.int32))
    rng = np.random.default_rng(2)
    P = (rng.standard_normal((200000, 3)) * 40).astype(np.float32)
    got = m.signed_distance(cu(P)).double().cpu().numpy()
    # the Hausdorff distance of mesh and sphere, from both sides: mesh samples against the sphere, sphere samples against the mesh
    u = rng.standard_normal((200000, 3))
    on_sphere = (u / np.linalg.norm(u, axis=1, keepdims=True) * r).astype(np.float32)
    h = max(deviation(m, lambda Q: sphere_sdf(Q, r), V), float(m.closest_points(cu(on_sphere))[0].max()))
    err = np.abs(got - sphere_sdf(P, r))
    print("fine sphere: %d faces, chord error %.4f, max |sdf - (|p| - r)| %.4f" % (F.shape[0], h, err.max()))
    assert h < 0.05 and err.max() <= 1.05 * h + 1e-4


# ------------------------------------------------------------------------------------------------ mesh distance
def small_spheres(r0, r1, n=24):
    c = (n / 2 - 0.7, n / 2 - 0.4, n / 2 - 0.9)
    a = mc_mesh(C.sphere_volume((n,) * 3, c, r0))
    b = mc_mesh(C.sphere_volume((n,) * 3, c, r1))
    return Mesh(cu(a[0]), cu(a[1], torch.int32)), Mesh(cu(b[0]), cu(b[1], torch.int32))


def test_mesh_distance_repeats_self_and_symmetry(cuda):
    a, b = small_spheres(8.0, 8.6)
    r1 = mesh_distance(a, b, nr_samples=200000, seed=3)
    r2 = mesh_distance(a, b, nr_samples=200000, seed=3)
    for k in ("accuracy", "completeness", "chamfer", "hausdorff"):
        assert r1[k] == r2[k]
    assert torch.equal(r1["dist_a_to_b"], r2["dist_a_to_b"]) and torch.equal(r1["dist_b_to_a"], r2["dist_b_to_a"])
    assert r1["dist_a_to_b"].shape == (200000,) and r1["chamfer"] == (r1["accuracy"] + r1["completeness"]) / 2
    sw = mesh_distance(b, a, nr_samples=200000, seed=3)
    assert sw["accuracy"] == r1["completeness"] and sw["completeness"] == r1["accuracy"] and sw["hausdorff"] == r1["hausdorff"]
    assert torch.equal(sw["dist_a_to_b"], r1["dist_b_to_a"])
    # a mesh against itself: the fp32 rounding of the sampled points (coordinates up to about 20, ulp 2e-6), and on marching-cubes
    # slivers at most about their width
    s = mesh_distance(a, a, nr_samples=200000, seed=3)
    print("self distance: chamfer %.3e, hausdorff %.3e" % (s["chamfer"], s["hausdorff"]))
    assert s["hausdorff"] < 1e-4 and s["chamfer"] < 2e-6
    # a different seed draws different samples
    assert mesh_distance(a, b, nr_samples=200000, seed=4)["accuracy"] != r1["accuracy"]


def test_samples_equal_the_oracle(cuda):
    a, _ = small_spheres(8.0, 8.6)
    pts, face = a._sample_surface("test", 50000, 11)
    V, F = a.V.cpu().numpy(), a.F.cpu().numpy()
    _, _, cdf = a._area_cdf("test")
    rp, rf = MD.sample_surface(V, F, cdf.cpu().numpy(), 50000, 11)
    assert np.array_equal(face.cpu().numpy(), rf) and np.array_equal(pts.cpu().numpy(), rp)
    p2, f2 = a._sample_surface("test", 1000, 11)
    assert torch.equal(p2, pts[:1000]) and torch.equal(f2, face[:1000])
    # the cdf: the fixed-point areas summed exactly, each face's share within 2^-60 of its fp64 area share
    p = V.astype(np.float64)[F]
    area = np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1) * 0.5
    c = cdf.cpu().numpy()
    assert torch.equal(cdf, a._area_cdf("test")[2]) and (np.diff(c) >= 0).all()
    share = np.diff(np.concatenate([[0.0], c])) / c[-1]
    assert np.abs(share - area / area.sum()).max() < 1e-12


def test_mesh_distance_against_the_fp64_oracle(cuda):
    a, b = small_spheres(7.0, 7.5, n=20)
    b.V = (b.V - b.V.mean(0)) @ cu(rotation(2).astype(np.float32)).T + b.V.mean(0) + 0.2
    N = 6000
    r = mesh_distance(a, b, nr_samples=N, seed=1)
    sa, _ = a._sample_surface("test", N, 1)
    sb, _ = b._sample_surface("test", N, 1)
    ref = MD.mesh_distance64(a.V.cpu().numpy(), a.F.cpu().numpy(), b.V.cpu().numpy(), b.F.cpu().numpy(), sa.cpu().numpy(),
                             sb.cpu().numpy())
    for k in ("accuracy", "completeness", "chamfer", "hausdorff"):
        assert abs(r[k] - ref[k]) <= 1e-3 * ref[k], (k, r[k], ref[k])


def test_concentric_spheres_are_delta_apart(cuda):
    a, b = small_spheres(20.0, 21.0, n=56)
    r = mesh_distance(a, b, nr_samples=500000)
    print("concentric spheres 20 / 21: %s" % {k: r[k] for k in ("accuracy", "completeness", "chamfer", "hausdorff")})
    for k in ("accuracy", "completeness", "chamfer"):
        assert abs(r[k] - 1.0) < 0.03, (k, r[k])
    assert abs(r["hausdorff"] - 1.0) < 0.15


# ------------------------------------------------------------------------------------------------ end to end: a fitted SDF against its mesh
# Bars from three H100 runs (H100 80GB HBM3, 700 W; the fit's float atomics make runs differ): (a) mean |learned sdf - signed_distance|
# measured 9.2e-4 to 1.1e-3, (b) chamfer distance of the mesh extracted at N = 256 measured 5.2e-4 to 8.0e-4 (Hausdorff 1.5e-3 to
# 1.7e-3). Each bar is about three times the largest value.
BAR_SDF, BAR_CHAMFER = 3e-3, 2.5e-3


def test_fitted_torus_against_its_mesh(cuda):
    from permuto_sdf_b200 import SurfaceFit
    from permuto_sdf_b200.mesh import extract_mesh_from_sdf_model
    N = 160
    lin = torch.linspace(-0.5, 0.5, N, device="cuda")
    grid = torch.stack(torch.meshgrid(lin, lin, lin, indexing="ij"), -1).reshape(-1, 3)
    q = torch.stack([grid[:, :2].norm(dim=-1) - 0.25, grid[:, 2]], -1)
    V, Fc = marching_cubes((q.norm(dim=-1) - 0.1).reshape(N, N, N).contiguous(), 0.0)
    mesh = Mesh(V, Fc)
    mesh.normalize_size()
    mesh.normalize_position()
    mesh.scale_mesh(0.6)
    mesh.recalculate_normals()
    mesh.upsample(1, True)
    f = SurfaceFit.from_mesh(mesh)
    f.enable_cuda_graph()
    f.fit(3000)
    g = torch.Generator(device="cuda").manual_seed(3)
    box = torch.rand(400000, 3, device="cuda", generator=g) - 0.5
    truth = mesh.signed_distance(box)
    near = truth.abs() < 0.05
    with torch.no_grad():
        learned = f.model_sdf.fused(box[near].contiguous(), f.iter_nr, with_gradient=False, with_geom=False)[0].view(-1)
    err = float((learned - truth[near]).abs().mean())
    extracted = extract_mesh_from_sdf_model(f.model_sdf, 256, -0.5, 0.5)
    r = mesh_distance(extracted, mesh, nr_samples=1_000_000)
    print("fitted torus: %d near points, mean |learned - signed_distance| %.3e; extracted %d faces, chamfer %.3e, accuracy %.3e, "
          "completeness %.3e, hausdorff %.3e" % (int(near.sum()), err, extracted.F.shape[0], r["chamfer"], r["accuracy"],
                                                 r["completeness"], r["hausdorff"]))
    assert err < BAR_SDF and r["chamfer"] < BAR_CHAMFER, (err, r["chamfer"])
