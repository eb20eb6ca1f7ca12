"""Mesh.winding_number and Mesh.signed_distance(sign="winding") on the GPU: the exact sum (beta = +inf) against the fp64 oracle
(oracle/winding.py) within the rounding bound of its fp32 terms; the far field (beta = 2) against the oracle within measured bars; the
same bits on every call, for any order of the points, and for a welded and an unwelded STL of one mesh; the winding sign against the
pseudonormal sign on closed meshes and against the oracle on open meshes and soups; and an SDF fitted to an open mesh checked against
the winding sign."""
import math

import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import winding as WN
from permuto_sdf_b200.mesh import Mesh, marching_cubes
from test_mesh_io_cpu import stl_binary
from test_mesh_raycast_gpu import cu, mc_mesh
from test_mesh_winding_cpu import uv_sphere

pytestmark = pytest.mark.gpu

# The far field at beta = 2 against the fp64 oracle over every mesh and point set of test_far_field_against_the_oracle, measured on an
# H100 80GB HBM3 (700 W): largest |w - w_exact| 3.9e-3 (torus, points 1e-3 off the surface), mean 6.6e-4. The bars are two and three
# times those.
BAR_MAX_BETA2, BAR_MEAN_BETA2 = 8e-3, 2e-3


def mesh_of(V, F):
    return Mesh(cu(V), cu(np.asarray(F, np.int32).reshape(-1, 3), torch.int32))


def cut_sphere():
    """a marching-cubes sphere with the cap z > 0.6 r removed: open, with one boundary loop"""
    V, F = mc_mesh(C.sphere_volume((30,) * 3, (14.3, 14.6, 14.1), 11.0))
    cz = V[F].mean(1)[:, 2] - 14.1
    return V, F[cz < 0.6 * 11.0]


def soup(seed, n=1500):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-1, 1, (n, 1, 3))
    return (c + rng.standard_normal((n, 3, 3)) * rng.uniform(0.01, 0.3, (n, 1, 1))).reshape(-1, 3).astype(np.float32), \
        np.arange(3 * n).reshape(-1, 3)


def degenerate():
    """a closed tetrahedron plus zero-area faces (collinear, repeated index, two equal corners under distinct indices)"""
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [2, 0, 0], [0, 0, 0], [0.5, 0.5, 0]], np.float32)
    F = [[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3], [0, 1, 4], [0, 0, 2], [3, 3, 3], [5, 0, 1], [1, 6, 2], [2, 5, 3]]
    return V, np.array(F)


MESHES = {
    "sphere": lambda: mc_mesh(C.sphere_volume((30,) * 3, (14.3, 14.6, 14.1), 11.0)),
    "torus": lambda: mc_mesh(C.torus_volume((40, 40, 20), (19.4, 19.7, 9.6), 13.0, 5.0)),
    "two_spheres": lambda: mc_mesh(C.two_spheres_volume((40, 24, 24), (12.0, 11.6, 11.8), (27.0, 11.6, 11.8), 7.5)),
    "cut_sphere": cut_sphere,
    "hemisphere": lambda: uv_sphere(12, 32, hemisphere=True),
    "soup": lambda: soup(0),
    "degenerate": degenerate,
    "one_face": lambda: (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), np.array([[0, 1, 2]])),
    "no_face": lambda: (np.zeros((3, 3), np.float32), np.zeros((0, 3), np.int64)),
}


def point_sets(V, F, seed=0, n=1500):
    """uniform over 1.5x the box, face points +- 1e-3 along the face normal, and the vertices"""
    rng = np.random.default_rng(seed)
    lo, hi = V.min(0), V.max(0)
    c, h = (lo + hi) / 2, (hi - lo) / 2 * 1.5 + 1e-3
    uni = rng.uniform(c - h, c + h, (n, 3))
    if len(F) == 0:
        return {"uniform": uni.astype(np.float32), "vertices": V.astype(np.float32)}
    t = V.astype(np.float64)[np.asarray(F)[rng.integers(0, len(F), n)]]
    b = rng.dirichlet((1, 1, 1), n)
    q = np.einsum("nk,nkd->nd", b, t)
    nrm = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    ln = np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm = np.where(ln > 0, nrm / np.where(ln > 0, ln, 1), 0)
    s = np.where(rng.random((n, 1)) < 0.5, 1e-3, -1e-3)
    return {"uniform": uni.astype(np.float32), "surface": (q + s * nrm).astype(np.float32), "vertices": V.astype(np.float32)}


def gpu_w(V, F, P, beta):
    return mesh_of(V, F).winding_number(cu(P), beta).cpu().numpy()


# ------------------------------------------------------------------------------------------------ exact sum == the oracle, to rounding
@pytest.mark.parametrize("name", list(MESHES))
def test_exact_sum_against_the_oracle(cuda, name):
    """beta = inf: every face's fp32 solid angle, summed in fp64 and rounded once. The oracle sums the fp64 solid angles of the same faces
    under the same skip rules, so they differ only by the rounding of the fp32 terms; WN.rounding_bound bounds that per point (first
    order in u = 2^-24: det within gamma_12 of its six products, den within gamma_20 of its terms, atan2 moved by at most the rounding box
    over its distance from the origin, or the whole 2 pi where the sign of det is undecided; plus atan2f's 4 ulp, the fp64 sum and the
    final fp32 rounding)."""
    V, F = MESHES[name]()
    for kind, P in point_sets(V, F).items():
        w = gpu_w(V, F, P, math.inf)
        ref = WN.winding_numbers(V, F, P)
        bound = WN.rounding_bound(V, F, P)
        err = np.abs(w.astype(np.float64) - ref)
        bad = np.flatnonzero(err > bound)
        assert bad.size == 0, (name, kind, bad.size, P[bad[:3]], w[bad[:3]], ref[bad[:3]], bound[bad[:3]])
        if len(F) == 0:
            assert (w == 0).all()


def test_known_values(cuda):
    V, F = uv_sphere(16, 32)
    inside = np.array([[0, 0, 0], [0.3, -0.2, 0.5], [0, 0, -0.9]], np.float32)
    outside = np.array([[2, 0, 0], [0, 0, 1.5], [-3, 4, 5]], np.float32)
    for beta, tol in ((math.inf, 1e-5), (2.0, BAR_MAX_BETA2)):
        w = gpu_w(V, F, np.concatenate([inside, outside]), beta)
        assert np.abs(w - [1, 1, 1, 0, 0, 0]).max() < tol, (beta, w)
        assert np.abs(gpu_w(V, F[:, ::-1], inside, beta) + 1).max() < tol
    Vh, Fh = uv_sphere(12, 32, hemisphere=True)
    assert abs(gpu_w(Vh, Fh, np.zeros((1, 3), np.float32), math.inf)[0] - 0.5) < 1e-6


# ------------------------------------------------------------------------------------------------ far field
def far_field_errors():
    errs, cases = [], []
    for name in ("sphere", "torus", "two_spheres", "cut_sphere", "hemisphere", "soup", "degenerate"):
        V, F = MESHES[name]()
        for kind, P in point_sets(V, F, seed=1).items():
            # points whose exact value is undecided by rounding (on a face's plane, inside the face: the sign of det is not known, and
            # the bound takes a whole 2 pi for that face) are left out; at such points w itself is not defined
            ok = WN.rounding_bound(V, F, P) < 0.1
            w = gpu_w(V, F, P[ok], 2.0).astype(np.float64)
            ref = WN.winding_numbers(V, F, P[ok])
            errs.append(np.abs(w - ref))
            cases.append((name, kind, w, ref))
    return errs, cases


def test_far_field_against_the_oracle(cuda):
    errs, cases = far_field_errors()
    e = np.concatenate(errs)
    print("beta = 2: max |w - w_exact| %.3e, mean %.3e over %d points; per case max: %s" % (
        e.max(), e.mean(), e.size, ", ".join("%s/%s %.2e (%d)" % (c[0], c[1], x.max(initial=0), x.size) for c, x in zip(cases, errs))))
    assert e.max() < BAR_MAX_BETA2 and e.mean() < BAR_MEAN_BETA2
    # the inside / outside decision agrees wherever the exact value is farther from 1/2 than the largest error
    for name, kind, w, ref in cases:
        sure = np.abs(ref - 0.5) > BAR_MAX_BETA2
        assert ((w > 0.5) == (ref > 0.5))[sure].all(), (name, kind)


# ------------------------------------------------------------------------------------------------ the same bits
def test_same_bits_on_every_call_and_for_any_point_order(cuda):
    V, F = MESHES["torus"]()
    m = mesh_of(V, F)
    P = cu(np.concatenate(list(point_sets(V, F, seed=2, n=20000).values())))
    perm = torch.randperm(P.shape[0], device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    for beta in (2.0, math.inf):
        a = m.winding_number(P, beta)
        assert torch.equal(a.view(torch.int32), m.winding_number(P, beta).view(torch.int32))
        assert torch.equal(a[perm].view(torch.int32), m.winding_number(P[perm].contiguous(), beta).view(torch.int32))


def test_welded_and_unwelded_stl_give_the_same_bits(cuda, tmp_path):
    V, F = cut_sphere()
    path = tmp_path / "cut.stl"
    path.write_bytes(stl_binary(V[F]))
    welded, soup_ = Mesh.load(path), Mesh.load(path, weld=False)
    assert welded.V.shape[0] < soup_.V.shape[0] and welded.F.shape == soup_.F.shape
    P = cu(np.concatenate(list(point_sets(V, F, seed=3).values())))
    for beta in (2.0, math.inf):
        a, b = welded.winding_number(P, beta), soup_.winding_number(P, beta)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), beta
    a, b = welded.signed_distance(P, sign="winding"), soup_.signed_distance(P, sign="winding")
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------------------------------------ signed_distance(sign="winding")
@pytest.mark.parametrize("name", ["sphere", "torus", "two_spheres"])
def test_winding_sign_on_closed_meshes(cuda, name):
    V, F = MESHES[name]()
    m = mesh_of(V, F)
    rng = np.random.default_rng(4)
    P = cu(np.concatenate(list(point_sets(V, F, seed=4, n=20000).values()) + [V + rng.normal(0, 0.3, V.shape).astype(np.float32)]))
    sd = m.signed_distance(P, sign="winding")
    pn = m.signed_distance(P)
    dist = m.closest_points(P)[0]
    assert torch.equal(sd.abs().view(torch.int32), dist.view(torch.int32))
    out = dist > 1e-3
    assert torch.equal(sd[out].view(torch.int32), pn[out].view(torch.int32))
    assert not bool((sd[dist == 0].view(torch.int32) != 0).any())             # +0 on the surface


@pytest.mark.parametrize("name", ["cut_sphere", "hemisphere", "soup", "degenerate", "no_face"])
def test_winding_sign_on_open_meshes_and_soups(cuda, name):
    V, F = MESHES[name]()
    m = mesh_of(V, F)
    P = np.concatenate(list(point_sets(V, F, seed=5).values()))
    sd = m.signed_distance(cu(P), sign="winding").cpu().numpy()
    dist = m.closest_points(cu(P))[0].cpu().numpy()
    assert (np.abs(sd).view(np.int32) == dist.view(np.int32)).all()
    ref = WN.winding_numbers(V, F, P)
    sure = (np.abs(ref - 0.5) > BAR_MAX_BETA2 + WN.rounding_bound(V, F, P)) & (dist > 0)
    assert ((sd < 0) == (ref > 0.5))[sure].all()
    if len(F) == 0:
        assert np.isposinf(sd).all()


# ------------------------------------------------------------------------------------------------ a fit to an open mesh
# Sign agreement of the fitted SDF with signed_distance(sign="winding") on the test's grid points, measured on an H100 80GB HBM3 (700 W):
# 0.9991 and 0.9989 of 60452 points (616 inside) on two runs. The bar is 0.98.
BAR_FIT_AGREEMENT = 0.98


def test_fit_to_a_cut_sphere_agrees_with_the_winding_sign(cuda):
    from permuto_sdf_b200 import SurfaceFit
    N = 96
    lin = torch.linspace(-0.5, 0.5, N, device="cuda")
    grid = torch.stack(torch.meshgrid(lin, lin, lin, indexing="ij"), -1).reshape(-1, 3)
    V, Fc = marching_cubes((grid.norm(dim=-1) - 0.3).reshape(N, N, N).contiguous(), 0.0)
    keep = V[Fc.long()].mean(1)[:, 2] < (N - 1) * (0.5 + 0.6 * 0.3)   # grid units: the cap above z = 0.6 r removed
    mesh = Mesh(V, Fc[keep].contiguous())
    mesh.remove_unreferenced_verts()
    mesh.normalize_size()
    mesh.normalize_position()
    mesh.scale_mesh(0.6)
    mesh.recalculate_normals()
    mesh.upsample(1, True)
    f = SurfaceFit.from_mesh(mesh)
    f.fit(400)
    g = torch.linspace(-0.45, 0.45, 40, device="cuda")
    P = torch.stack(torch.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).contiguous()
    w = mesh.winding_number(P, math.inf)
    sd = mesh.signed_distance(P, sign="winding")
    sel = ((w - 0.5).abs() > 0.25) & (sd.abs() > 0.05)
    with torch.no_grad():
        learned = f.model_sdf.fused(P[sel].contiguous(), f.iter_nr, with_gradient=False, with_geom=False)[0].view(-1)
    agree = float(((learned < 0) == (sd[sel] < 0)).float().mean())
    print("fit to a cut sphere: %d grid points, %d inside, sign agreement %.4f" % (int(sel.sum()), int((sd[sel] < 0).sum()), agree))
    assert int((sd[sel] < 0).sum()) > 100 and agree > BAR_FIT_AGREEMENT
