"""Marching cubes on the GPU (csrc/marching_cubes.cu, permuto_sdf_b200/mesh.py): bit for bit and in order against the numpy oracle on the
256 single-cell volumes, analytic, random and degenerate volumes; independence of the slab split and of the run; extract_mesh_from_sdf_model
against the dense grid of the same fused forward; meshes of trained models; a grid with more than 2^31 cells; edge cases and side effects."""
import math

import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import marching_cubes as M

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _reduction_mode_off_after(cuda):
    """SurfaceFit(deterministic=True) switches the device's mode on; later tests start from the default"""
    yield
    from permuto_sdf_b200 import call
    call("psdf_set_deterministic", 0, 0, 0)


def same_bits(gpu, ref):
    """gpu (verts, faces) equal the oracle's bit for bit and in order"""
    V, F = gpu
    V, F = V.cpu().numpy(), F.cpu().numpy()
    return V.shape == ref[0].shape and F.shape == ref[1].shape and np.array_equal(V.view(np.int32), ref[0].view(np.int32)) and \
        np.array_equal(F, ref[1])


def rescale(V, N, min_val, max_val):
    """the reference's rescale (sdf_utils.py:283) in float32"""
    return V / np.float32(N - 1) * np.float32(max_val - min_val) + np.float32(min_val)


# ------------------------------------------------------------------------------------------------ tables and volumes vs the oracle
def test_single_cell_volumes_match_oracle(cuda):
    from permuto_sdf_b200 import marching_cubes
    for cfg in range(256):
        v = M.single_cell_volume(cfg, inside=-0.75, outside=0.5)
        got = marching_cubes(torch.from_numpy(v).cuda())
        assert same_bits(got, M.marching_cubes(v, 0.0)), cfg
        assert got[1].shape[0] == len(M.TABLE[cfg])


VOLUMES = {
    "sphere": lambda: (C.sphere_volume((72, 80, 64), (35.3, 40.1, 31.7), 25.0), 0.0),
    "torus": lambda: (C.torus_volume((64, 66, 24), (31.6, 32.2, 11.4), 20.0, 7.0), 0.0),
    "touching_spheres": lambda: (C.two_spheres_volume((90, 60, 60), (29.5, 30.2, 29.8), (59.5, 30.2, 29.8), 15.0), 0.0),
    "sphere_threshold": lambda: (C.sphere_volume((67, 45, 131), (33.1, 22.4, 60.2), 12.0), 3.7),
    "random": lambda: (C.random_field((96, 80, 71), seed=3), 0.0),
    "random_open_threshold": lambda: (np.random.default_rng(4).standard_normal((37, 29, 53)).astype(np.float32), 0.21),
    "axis0_len2": lambda: (np.random.default_rng(5).standard_normal((2, 37, 45)).astype(np.float32), -0.1),
    "axis1_len2": lambda: (np.random.default_rng(6).standard_normal((41, 2, 19)).astype(np.float32), 0.0),
    "axis2_len2": lambda: (np.random.default_rng(7).standard_normal((23, 31, 2)).astype(np.float32), 0.3),
    "all_len2": lambda: (np.random.default_rng(8).standard_normal((2, 2, 2)).astype(np.float32), 0.0),
    "exact_threshold": lambda: (C.pad_outside(np.random.default_rng(0).integers(-1, 2, (20, 17, 23)).astype(np.float32)), 0.0),
    "checkerboard": lambda: (C.pad_outside(((np.indices((12, 13, 11)).sum(0)) % 2 * 2 - 1).astype(np.float32)), 0.0),
}


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_volumes_match_oracle_bit_for_bit(cuda, name):
    from permuto_sdf_b200 import marching_cubes
    vol, thr = VOLUMES[name]()
    ref = M.marching_cubes(vol, thr)
    got = marching_cubes(torch.from_numpy(vol).cuda(), thr)
    assert got[0].dtype == torch.float32 and got[1].dtype == torch.int32
    assert same_bits(got, ref), (name, got[0].shape, ref[0].shape, got[1].shape, ref[1].shape)


def test_slab_split_and_run_do_not_change_the_result(cuda):
    from permuto_sdf_b200.mesh import _marching_cubes
    for vol, thr in (VOLUMES["random"](), VOLUMES["sphere_threshold"]()):
        v = torch.from_numpy(vol).cuda()
        runs = [_marching_cubes(v, thr, s) for s in (1, 7, vol.shape[0] - 1, None, 1, 7)]
        for V, F in runs[1:]:
            assert torch.equal(V.view(torch.int32), runs[0][0].view(torch.int32)) and torch.equal(F, runs[0][1])


def test_refusals(cuda):
    from permuto_sdf_b200 import marching_cubes
    with pytest.raises(RuntimeError, match=">= 2"):
        marching_cubes(torch.zeros(1, 5, 5, device="cuda"))
    with pytest.raises(RuntimeError, match="shape"):
        marching_cubes(torch.zeros(5, 5, device="cuda"))
    with pytest.raises(RuntimeError, match="finite"):
        marching_cubes(torch.zeros(3, 3, 3, device="cuda"), float("nan"))


# ------------------------------------------------------------------------------------------------ models
@pytest.fixture(scope="module")
def sphere_trainer(cuda):
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=128, nr_images=4, seed=5, optimizer="fused")
    tr.set_analytic_scene()
    tr.fit_sphere()
    torch.cuda.synchronize()
    return tr


@pytest.fixture(scope="module")
def surface_fit(cuda):
    """the convergence run of test_surface_fit_gpu on its sphere cloud"""
    from permuto_sdf_b200 import SurfaceFit
    g = torch.Generator(device="cuda").manual_seed(1)
    d = torch.nn.functional.normalize(torch.randn(200000, 3, device="cuda", generator=g), dim=-1)
    f = SurfaceFit((torch.tensor([0.1, -0.05, 0.08], device="cuda") + 0.3 * d).contiguous(), d.contiguous())
    f.enable_cuda_graph()
    f.fit(3000)
    torch.cuda.synchronize()
    return f


def test_extraction_equals_dense_grid(sphere_trainer):
    from permuto_sdf_b200 import extract_mesh_from_sdf_model, marching_cubes
    from permuto_sdf_b200.permuto_sdf import PermutoSDF
    m = sphere_trainer.model_sdf
    N, lo, hi = 160, -0.5, 0.5
    mesh = extract_mesh_from_sdf_model(m, N, lo, hi)
    with torch.no_grad():
        pts = PermutoSDF.meshgrid3d(lo, hi, N).reshape(-1, 3).contiguous()
        dense = m.fused(pts, 9999999, with_gradient=False, with_geom=False)[0].view(N, N, N)
    V, F = marching_cubes(dense)
    assert len(F) > 1000
    assert np.array_equal(rescale(V.cpu().numpy(), N, lo, hi).view(np.int32), mesh.V.cpu().numpy().view(np.int32))
    assert torch.equal(F, mesh.F)
    Vo, Fo = M.marching_cubes(dense.cpu().numpy(), 0.0)
    assert np.array_equal(rescale(Vo, N, lo, hi).view(np.int32), mesh.V.cpu().numpy().view(np.int32))
    assert np.array_equal(Fo, mesh.F.cpu().numpy())


def check_sphere_mesh(mesh, center, radius, tol, cos_mean=0.995, cos_min=0.9):
    V, F = mesh.V.cpu().numpy(), mesh.F.cpu().numpy()
    assert C.closed_and_oriented(F, len(V)) and C.euler_characteristic(F) == 2
    rel = V - np.asarray(center, dtype=np.float32)
    r = np.linalg.norm(rel, axis=1)
    assert np.abs(r - radius).max() < tol and np.abs(r - radius).mean() < 0.003, (np.abs(r - radius).max(), np.abs(r - radius).mean())
    cos = (mesh.NV.cpu().numpy() * rel).sum(1) / r
    assert cos.mean() > cos_mean and cos.min() > cos_min, (cos.mean(), cos.min())
    assert abs(C.signed_volume(V, F) / (4 / 3 * math.pi * radius ** 3) - 1) < 0.02


def test_trained_sphere_fit_mesh(sphere_trainer):
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    mesh = extract_mesh_from_sdf_model(sphere_trainer.model_sdf, 256, -0.5, 0.5)
    # the fit draws its points inside the bounding sphere (radius 0.5); towards the grid's corners the network has zero crossings of its own
    mesh.remove_marked_vertices(mesh.V.norm(dim=1) < 0.42, True)
    # the small fitted model (8 levels) is off by up to ~1 % of the radius, and its gradient by up to ~35 degrees at a few vertices
    check_sphere_mesh(mesh, (0.0, 0.0, 0.0), 0.3, 0.02, cos_mean=0.99, cos_min=0.7)


def test_surface_fit_mesh_and_cropping(surface_fit):
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    m = surface_fit.model_sdf
    mesh = extract_mesh_from_sdf_model(m, 256, -0.5, 0.5)
    check_sphere_mesh(mesh, (0.1, -0.05, 0.08), 0.3, 0.01)
    # crop with the model's boundary primitive, as create_my_meshes.py:72-74 does
    full = extract_mesh_from_sdf_model(m, 96, -0.6, 0.6, threshold=0.05)
    inside = m.boundary_primitive.check_point_inside_primitive(full.V).view(-1)
    assert int(inside.sum()) > 0
    V0, F0 = full.V.clone(), full.F.clone()
    full.remove_marked_vertices(inside, True)
    assert torch.equal(full.V, V0[inside]) and bool(m.boundary_primitive.check_point_inside_primitive(full.V).all())
    keep_face = inside[F0.long()].all(1)
    new_id = torch.cumsum(inside.long(), 0) - 1
    assert torch.equal(full.F, new_id[F0[keep_face].long()].int())


def test_large_grid_streams(sphere_trainer):
    """N = 1300: 2.2e9 grid points and cells, more than 2^31; the dense volume would be 8.8 GB"""
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    N = 1300
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    mesh = extract_mesh_from_sdf_model(sphere_trainer.model_sdf, N, -0.5, 0.5)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("N = %d: %d vertices, %d faces, peak %.0f MB" % (N, mesh.V.shape[0], mesh.F.shape[0], peak / 2 ** 20))
    assert peak < N ** 3 * 4 / 8
    r = mesh.V.norm(dim=1)
    near = r < 0.42                     # the fitted sphere; beyond the bounding sphere the network has zero crossings of its own
    assert int(near.sum()) > 1000000 and float((r[near] - 0.3).abs().max()) < 0.02
    F = mesh.F
    assert int(F.min()) == 0 and int(F.max()) == mesh.V.shape[0] - 1
    assert torch.unique(F).numel() == mesh.V.shape[0]


def test_threshold_outside_range_and_open_surface(sphere_trainer):
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    m = sphere_trainer.model_sdf
    empty = extract_mesh_from_sdf_model(m, 64, -0.5, 0.5, threshold=100.0)
    assert empty.V.shape == (0, 3) and empty.F.shape == (0, 3) and empty.NV.shape == (0, 3)
    cut = extract_mesh_from_sdf_model(m, 80, -0.2, 0.25)          # the r = 0.3 sphere crosses the grid's faces
    F = cut.F.cpu().numpy()
    assert len(F) > 0 and F.max() < cut.V.shape[0] and not C.closed_and_oriented(F, cut.V.shape[0])
    assert float(cut.V.abs().max()) <= 0.25


def test_no_side_effects(sphere_trainer):
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    from permuto_sdf_b200.models import SDF
    from permuto_sdf_b200.permuto_sdf import Sphere
    m = sphere_trainer.model_sdf
    before = {k: v.clone() for k, v in m.state_dict().items()}
    for training in (True, False):
        m.train(training)
        m.last_iter_nr = 123
        extract_mesh_from_sdf_model(m, 48, -0.5, 0.5, iter_nr=7)
        assert m.training == training and m.last_iter_nr == 123
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k
    bare = SDF(3, Sphere(0.5, [0, 0, 0]), 0, 100, nr_levels=8, capacity=2 ** 14, hidden=64).cuda()
    mesh = extract_mesh_from_sdf_model(bare, 48, -0.5, 0.5, threshold=0.01)
    assert getattr(bare, "fused", None) is None and mesh.V.dtype == torch.float32
