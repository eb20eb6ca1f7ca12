"""Meshes from a trained NeRF (csrc/fused_bg.cu's density-only k_bg_fused<3, true>, FusedNerfHash.density, NerfHash.get_only_density,
mesh.extract_mesh_from_density_model):
  * psdf_nerf_density_forward bit-identical to the density of psdf_nerf_fused_forward(3, ...) at the shape limits, rows >= N untouched,
    and against the fp64 reference with the bounds of test_fused_forward_fp64_gpu.py;
  * get_only_density: fused against per-op inside the coarse-to-fine ramp, against the reference's own outputs, no last_iter_nr;
  * extraction bit for bit against the dense grid of the full forward meshed by marching_cubes and the numpy oracle, for any slab split;
    normals bit for bit against central differences of the full forward;
  * the mesh of a trained NeRF of the shaded sphere; edge cases, refusals and side effects."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import backward_fp64 as R
from oracle import marching_cubes as M
from test_fused_backward_fp64_gpu import cu, positions, window
from test_fused_forward_fp64_gpu import check, guarded, n_spec, rows
from test_nerf_train_gpu import FWD_CASES, _bg_weights, _blob

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(autouse=True)
def _deterministic_mode_off_afterwards():
    """NerfTrainer(deterministic=True) switches the device's deterministic mode on; later tests start without it"""
    yield
    from permuto_sdf_b200._lib import call
    call("psdf_set_deterministic", 0, 0, 0)


# ------------------------------------------------------------------------------------------------ the kernel
def _inputs(L, n, T, seed):
    g = torch.Generator().manual_seed(seed)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    W, b = _bg_weights(L, g)
    pos = positions("uniform", n, g, D=3)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    return lat, shift, W, b, pos, dirs


@pytest.mark.parametrize("L,N", FWD_CASES, ids=["L%d-N%s" % c for c in FWD_CASES])
def test_density_kernel_equals_full_forward(cuda, L, N):
    from permuto_sdf_b200._lib import call
    n, T = n_spec(N), 2 ** 16
    lat, shift, W, b, pos, dirs = _inputs(L, n, T, L * 100 + n % 97 + 1)
    blob = _blob(L, W, b)
    common = (n, L, T, cu(pos))
    enc = (lat.cuda(), R.level_scales(L, 3).cuda(), shift.cuda(), window(L, "mid").cuda(), 1.0, blob)
    rgb, full = torch.empty(n, 3, device="cuda"), guarded(n, 0)
    call("psdf_nerf_fused_forward", 3, *common, cu(dirs), *enc, rgb, full)
    den = guarded(n, 0)
    call("psdf_nerf_density_forward", *common, *enc, den)
    torch.cuda.synchronize()
    a, b_ = rows(full, n, "density"), rows(den, n, "density only")
    assert torch.equal(a.view(torch.int32), b_.view(torch.int32)), int((a != b_).sum())


def test_density_kernel_matches_fp64(cuda):
    from permuto_sdf_b200._lib import call
    L, n, T = 24, n_spec("2*128sms+5"), 2 ** 16
    lat, shift, W, b, pos, dirs = _inputs(L, n, T, 5)
    scale, w = R.level_scales(L, 3), window(L, "mid")
    ref = R.bg_forward_reference(pos, dirs, lat, scale, shift, w, 1.0, W, b, device="cuda")
    den = guarded(n, 0)
    call("psdf_nerf_density_forward", n, L, T, cu(pos), lat.cuda(), scale.cuda(), shift.cuda(), w.cuda(), 1.0, _blob(L, W, b), den)
    torch.cuda.synchronize()
    check("density L%d N%d" % (L, n), "nerf3_density", "density", rows(den, n, "density"), ref["density"], ref["A_density"])


def test_density_kernel_limits(cuda):
    from permuto_sdf_b200._lib import call
    L, T = 8, 2 ** 10
    lat, shift, W, b, pos, _ = _inputs(L, 4, T, 9)
    enc = (lat.cuda(), R.level_scales(L, 3).cuda(), shift.cuda(), window(L, "open").cuda(), 1.0, _blob(L, W, b))
    den = guarded(0, 0)
    call("psdf_nerf_density_forward", 0, L, T, cu(pos), *enc, den)           # N == 0: nothing written
    torch.cuda.synchronize()
    rows(den, 0, "density")
    for bad in ((4, 6, T), (4, 32, T), (-1, L, T), (4, L, 0)):
        with pytest.raises(RuntimeError, match="failed"):
            call("psdf_nerf_density_forward", bad[0], bad[1], bad[2], cu(pos), *enc, den)


# ------------------------------------------------------------------------------------------------ get_only_density
def _nerf(in_channels=3, c2f=10000, L=24, T=2 ** 16, seed=3):
    from permuto_sdf_b200.models import NerfHash
    from permuto_sdf_b200.permuto_sdf import Sphere
    torch.manual_seed(seed)
    m = NerfHash(in_channels, Sphere(0.5, [0, 0, 0]), c2f, L, T).cuda()
    with torch.no_grad():
        m.encoding.lattice_values.uniform_(-0.3, 0.3)
        m.mlp_feat_and_density[-1].bias[0] += 1.0
    return m


def test_get_only_density_fused_matches_per_op(cuda):
    from permuto_sdf_b200.models import map_range_val
    m = _nerf()
    pts = (torch.rand(3000 + 77, 3, device="cuda") - 0.5)
    m.last_iter_nr = 42
    with torch.no_grad():
        ref = m.get_only_density(pts, 3000)             # per-op: fused not enabled
    assert m.last_iter_nr == 42 and m.fused is None
    m.enable_fused()
    got = m.get_only_density(pts.view(1, -1, 3), 3000)     # reshaped to [-1, 3] as the reference does
    assert m.last_iter_nr == 42 and got.shape == (pts.shape[0], 1) and not got.requires_grad
    w = m.c2f(map_range_val(3000, 0.0, m.nr_iters_for_c2f, 0.3, 1.0)).view(-1)
    assert bool(((w > 0) & (w < 1)).any())               # inside the coarse-to-fine ramp
    err = float(((got - ref).abs() / ref.abs().clamp(min=1e-6)).max())
    assert err <= 1e-4, err
    full = m.fused(pts, torch.zeros_like(pts), 3000)[1]
    assert torch.equal(got, full)


def test_get_only_density_on_the_reference_fixture(cuda):
    """tests/golden/refpy_golden_nerf.npz: the reference's NerfHash(3) density at the foreground samples, iteration 5000"""
    from permuto_sdf_b200.nerf_train import NerfTrainer
    from test_refpy_golden_gpu import load, rel
    G = dict(np.load(os.path.join(HERE, "golden", "refpy_golden_nerf.npz")))
    tr = NerfTrainer(4, False)
    load(tr.model, G, "fg.", 21)
    pos = torch.from_numpy(np.ascontiguousarray(G["in.fg_pos"])).cuda()
    tr.model.last_iter_nr = 7
    fused = tr.model.get_only_density(pos, 5000)
    fb, tr.model.fused = tr.model.fused, None
    with torch.no_grad():
        per_op = tr.model.get_only_density(pos, 5000)
    tr.model.fused = fb
    assert tr.model.last_iter_nr == 7
    assert rel(fused, G["nomask.density"]) < 1e-4 and rel(per_op, G["nomask.density"]) < 1e-4


def test_density_refuses_four_d(cuda):
    m = _nerf(4, L=8, T=2 ** 10)
    fb = m.enable_fused()
    with pytest.raises(RuntimeError, match="pos_dim"):
        fb.density(torch.zeros(5, 4, device="cuda"), 0)


# ------------------------------------------------------------------------------------------------ a trained NeRF
# the iso-level of the trained NeRF's meshes: the tightest outer hull of 5, 10, 15 and 20 (see test_trained_nerf_mesh)
THR = 20.0


@pytest.fixture(scope="module")
def trained(cuda):
    """the convergence run of test_nerf_train_gpu: NerfTrainer(9, with_mask=True), 1500 iterations on the shaded sphere (radius 0.3)"""
    import bench
    from permuto_sdf_b200.nerf_train import NerfTrainer
    reel = bench.analytic_reel(9, 60, 80, 100.0, torch.device("cuda"))
    tr = NerfTrainer(9, True)
    g = torch.Generator().manual_seed(5)
    for _ in range(1500):
        pix = torch.randint(0, 60 * 80, (512,), generator=g).to(torch.int32)
        img = torch.randint(0, 8, (512,), generator=g).to(torch.int32)
        tr.step_from_reel(reel, pix, img)
    torch.cuda.synchronize()
    return tr


def rescale(V, N, lo, hi):
    return V / np.float32(N - 1) * np.float32(hi - lo) + np.float32(lo)


def _full_density(m, pts, it=9999999):
    return m.fused(pts.contiguous(), torch.zeros_like(pts), it)[1]


def test_extraction_equals_dense_grid(trained, monkeypatch):
    from permuto_sdf_b200 import extract_mesh_from_density_model, marching_cubes, mesh as mesh_mod
    from permuto_sdf_b200.permuto_sdf import PermutoSDF
    m = trained.model
    N, lo, hi = 112, -0.5, 0.5
    mesh = extract_mesh_from_density_model(m, N, lo, hi, threshold=THR)
    with torch.no_grad():
        dense = _full_density(m, PermutoSDF.meshgrid3d(lo, hi, N).reshape(-1, 3)).view(N, N, N)
    V, F = marching_cubes(-dense, -THR)
    assert len(F) > 1000
    Vm = mesh.V.cpu().numpy()
    assert np.array_equal(rescale(V.cpu().numpy(), N, lo, hi).view(np.int32), Vm.view(np.int32)) and torch.equal(F, mesh.F)
    Vo, Fo = M.marching_cubes((-dense).cpu().numpy(), -THR)
    assert np.array_equal(rescale(Vo, N, lo, hi).view(np.int32), Vm.view(np.int32)) and np.array_equal(Fo, mesh.F.cpu().numpy())
    # normals: central differences of the full forward at the same offset points
    h = float(np.float32(hi - lo) / np.float32(N - 1))
    with torch.no_grad():
        d = [[_full_density(m, mesh.V - s * h * torch.eye(3, device="cuda")[i]).view(-1) for i in range(3)] for s in (1, -1)]
    nv = torch.nn.functional.normalize(torch.stack(d[0], 1) - torch.stack(d[1], 1), dim=1)
    assert torch.equal(nv.view(torch.int32), mesh.NV.view(torch.int32))
    # several slabs, and normals in several chunks: the same bits
    monkeypatch.setattr(mesh_mod, "_SLAB_POINTS", N * N * 5 + 17)
    small = extract_mesh_from_density_model(m, N, lo, hi, threshold=THR)
    for a, b in ((small.V, mesh.V), (small.NV, mesh.NV)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.equal(small.F, mesh.F)


def _fibonacci_directions(n):
    i = torch.arange(n, dtype=torch.float64) + 0.5
    phi, th = torch.acos(1 - 2 * i / n), math.pi * (1 + 5 ** 0.5) * i
    return torch.stack([torch.cos(th) * torch.sin(phi), torch.sin(th) * torch.sin(phi), torch.cos(phi)], 1).float().cuda()


def test_trained_nerf_mesh(trained):
    """The density of the trained NeRF is ~25-40 inside the sphere (with scatter) and ~0 outside r = 0.32, so the mesh has the sphere as
    its outer hull plus surfaces of its own inside (the interior is never seen) and a few floaters. Measured on the outer hull: the
    outermost vertex in each of 2000 direction bins. Measured on an H100 80GB HBM3 (700 W), two runs at threshold 20: median |r - 0.3|
    of the hull 0.0058-0.0061, 92 % of the bins within 0.03 of 0.3, the hull normals' cosine with the radial direction median
    0.930-0.932 and mean 0.856-0.863. Bounds: 0.015, 85 %, 0.88 and 0.8."""
    from permuto_sdf_b200 import extract_mesh_from_density_model
    m = trained.model
    mesh = extract_mesh_from_density_model(m, 128, -0.5, 0.5, threshold=THR)
    mesh.remove_marked_vertices(m.boundary_primitive.check_point_inside_primitive(mesh.V).view(-1), True)
    V, NV = mesh.V, mesh.NV
    r = V.norm(dim=1)
    nb = 2000
    b = ((V / r[:, None]) @ _fibonacci_directions(nb).t()).argmax(1)
    hull = torch.zeros(nb, device="cuda").scatter_reduce(0, b, r, "amax", include_self=False)
    top = r == hull[b]
    cos = (NV[top] * V[top]).sum(1) / r[top]
    dev = (hull[torch.unique(b)] - 0.3).abs()
    print("\nthreshold %g: %d vertices, hull median |r - 0.3| %.4f, within 0.03 %.3f; hull cos median %.4f mean %.4f" % (
        THR, V.shape[0], float(dev.median()), float((dev < 0.03).float().mean()), float(cos.median()), float(cos.mean())))
    assert torch.unique(b).numel() == nb
    assert float(dev.median()) < 0.015 and float((dev < 0.03).float().mean()) > 0.85
    assert float(cos.median()) > 0.88 and float(cos.mean()) > 0.8


# ------------------------------------------------------------------------------------------------ edge cases
def test_threshold_above_the_field_and_open_surface(trained):
    import mesh_checks as C
    from permuto_sdf_b200 import extract_mesh_from_density_model
    m = trained.model
    empty = extract_mesh_from_density_model(m, 48, -0.5, 0.5, threshold=1e30)
    assert empty.V.shape == (0, 3) and empty.F.shape == (0, 3) and empty.NV.shape == (0, 3)
    cut = extract_mesh_from_density_model(m, 80, -0.2, 0.25, threshold=THR)      # the r = 0.3 sphere crosses the grid's faces
    F = cut.F.cpu().numpy()
    assert len(F) > 0 and F.max() < cut.V.shape[0] and not C.closed_and_oriented(F, cut.V.shape[0])
    assert float(cut.V.abs().max()) <= 0.25


def test_refusals(cuda):
    from permuto_sdf_b200 import extract_mesh_from_density_model
    m = _nerf(L=8, T=2 ** 10)
    with pytest.raises(RuntimeError, match="in_channels 4"):
        extract_mesh_from_density_model(_nerf(4, L=8, T=2 ** 10), 16, -0.5, 0.5)
    with pytest.raises(RuntimeError, match=">= 2"):
        extract_mesh_from_density_model(m, 1, -0.5, 0.5)
    for bad in ((float("nan"), 0.5, 0.0), (-0.5, float("inf"), 0.0), (-0.5, 0.5, float("nan"))):
        with pytest.raises(RuntimeError, match="finite"):
            extract_mesh_from_density_model(m, 16, bad[0], bad[1], threshold=bad[2])


def test_no_side_effects(trained):
    from permuto_sdf_b200 import extract_mesh_from_density_model
    m = trained.model
    before = {k: v.clone() for k, v in m.state_dict().items()}
    for training in (True, False):
        m.train(training)
        m.last_iter_nr = 123
        extract_mesh_from_density_model(m, 48, -0.5, 0.5, threshold=THR, iter_nr=7)
        assert m.training == training and m.last_iter_nr == 123
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k
    bare = _nerf(L=8, T=2 ** 10)
    bare.last_iter_nr = 5
    mesh = extract_mesh_from_density_model(bare, 48, -0.5, 0.5, threshold=1.0)
    assert bare.fused is None and bare.last_iter_nr == 5 and mesh.V.dtype == torch.float32 and mesh.NV.shape == mesh.V.shape
    assert math.isfinite(float(mesh.NV.sum()))
