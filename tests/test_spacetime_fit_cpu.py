"""Host logic of SpaceTimeFit and the space-time SDF without a device: the refusals of the constructor and of step() with their reasons,
the refusal of the fused training pair for a D = 4 SDF, and the fp64 reference at D = 4 (spatial tangents, upstream g_grad padded with a
zero time column) against fp64 autograd through the whole forward."""
import pytest
import torch

from oracle import backward_fp64 as R
from permuto_sdf_b200.surface_fit import SpaceTimeFit, SurfaceFit


def rel(a, b):
    a, b = torch.as_tensor(a).double().reshape(-1), torch.as_tensor(b).double().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


@pytest.mark.parametrize("points, normals, reason", [
    (torch.zeros(10, 3), torch.zeros(10, 3), r"SpaceTimeFit: points should have shape \[P,4\]"),
    (torch.zeros(10, 4), torch.zeros(10, 4), r"SpaceTimeFit: normals should have shape \[P,3\]"),
    (torch.zeros(10, 4, dtype=torch.float64), torch.zeros(10, 3), "points must be float32"),
    (torch.zeros(10, 4), torch.zeros(9, 3), "10 points but 9 normals"),
    (torch.zeros(0, 4), torch.zeros(0, 3), "point cloud is empty"),
    (torch.empty(2 ** 29, 4, device="meta"), torch.empty(2 ** 29, 3, device="meta"), r"32-bit row indexing takes \(at most 536870911\)"),
    (torch.zeros(10, 4), torch.zeros(10, 3), "must be on a CUDA device"),
])
def test_constructor_refusals(points, normals, reason):
    with pytest.raises(RuntimeError, match=reason):
        SpaceTimeFit(points, normals)


def test_surface_fit_still_refuses_space_time_points():
    with pytest.raises(RuntimeError, match=r"SurfaceFit: points should have shape \[P,3\]"):
        SurfaceFit(torch.zeros(10, 4), torch.zeros(10, 3))


@pytest.mark.parametrize("ns, no, reason", [(0, 3000, "SpaceTimeFit.step: needs at least one surface and one box point"),
                                            (3000, 0, "at least one surface"), (2 ** 28, 2 ** 28, "32-bit row indexing")])
def test_step_refusals(ns, no, reason):
    fit = SpaceTimeFit.__new__(SpaceTimeFit)          # no model: the counts are checked before anything runs
    with pytest.raises(RuntimeError, match=reason):
        fit.step(ns, no)
    with pytest.raises(RuntimeError, match=reason):
        fit.fit(3, ns, no)


def test_defaults_are_those_of_train_4d_sdf():
    import inspect
    sig = inspect.signature(SpaceTimeFit.__init__).parameters
    assert sig["nr_levels"].default == 24 and sig["capacity"].default == 2 ** 18 and sig["hidden"].default == 32
    assert sig["nr_iters_for_c2f"].default == 3000 and sig["lr"].default == 1e-3
    assert tuple(sig["box_size"].default) == (1, 1, 1) and tuple(sig["box_translation"].default) == (0, 0, 0)
    step = inspect.signature(SpaceTimeFit.step).parameters
    assert step["nr_surface"].default == 3000 and step["nr_offsurface"].default == 3000


def test_fused_training_is_refused_for_a_space_time_sdf():
    from permuto_sdf_b200.models import SDF
    m = SDF(4, None, 0, 3000, nr_levels=4, capacity=2 ** 10, hidden=16)
    with pytest.raises(RuntimeError, match=r"in_channels 4; get_sdf_and_gradient returns the \[N,4\] gradient including d sdf / dt"):
        m.enable_fused_training()
    assert not getattr(m, "fused_training", False) and getattr(m, "fused", None) is None
    # the per-op autograd path keeps serving the reference's call: the [N,4] gradient
    m.forward = lambda p, it: ((p[:, :3] ** 2).sum(1, keepdim=True) + p[:, 3:] * 0.5, None)
    p = torch.rand(5, 4)
    _, g, _ = m.get_sdf_and_gradient(p, 0)
    assert g.shape == (5, 4) and torch.allclose(g[:, 3], torch.full((5,), 0.5))


def _case4(N=300, L=8, T=2 ** 10, hidden=32, out_dim=9, seed=0):
    g = torch.Generator().manual_seed(seed)
    pos = torch.cat([(torch.rand(N, 3, generator=g) - 0.5) * 0.9, torch.rand(N, 1, generator=g)], 1)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 4, generator=g) * 10
    dims = [2 * L + 4, hidden, hidden, hidden, out_dim]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    up = (torch.randn(N, generator=g), torch.randn(N, 3, generator=g), torch.randn(N, out_dim - 1, generator=g))
    return pos, lat, R.level_scales(L, 4), shift, R.window_of(L, 0.6), W, b, up


@pytest.mark.parametrize("out_dim", [1, 9])
def test_d4_reference_with_spatial_upstream_matches_double_backward(out_dim):
    """the kernels' backward at D = 4: tangent along (g_grad, 0). The explicit reference and fp64 autograd of
    <g_grad, d sdf / d(x, y, z)> agree to 1e-12"""
    pos, lat, scale, shift, win, W, b, (gs, gg, gm) = _case4(out_dim=out_dim, seed=out_dim)
    gm = gm if out_dim > 1 else None
    gg4 = torch.cat([gg, torch.zeros(gg.shape[0], 1)], 1)
    ref = R.sdf_reference(pos, lat, scale, shift, win, 1e-3, W, b, gs, gg4, gm)
    lg, gW, gb, _ = R.sdf_autograd(pos, lat, scale, shift, win, 1e-3, W, b, gs, gg4, gm)
    assert rel(R.dense_lattice(ref["lattice"]), lg) < 1e-12
    for l in range(4):
        assert rel(ref["W"][l], gW[l]) < 1e-12 and rel(ref["b"][l], gb[l]) < 1e-12, l
    # the padded time column is what makes this the spatial directional derivative: a non-zero time upstream changes the result
    gt = gg4.clone()
    gt[:, 3] = 1.0
    lt = R.sdf_autograd(pos, lat, scale, shift, win, 1e-3, W, b, gs, gt, gm)[0]
    assert rel(lt, lg) > 1e-6


def test_d4_forward_reference_spatial_tangents_match_autograd():
    """the forward reference's tangent streams at D = 4 against fp64 autograd of sdf wrt the position; columns 0..2 are what the kernels
    return"""
    pos, lat, scale, shift, win, W, b, _ = _case4(N=200, L=4, T=5003, hidden=16, out_dim=5, seed=3)
    ref = R.sdf_forward_reference(pos, lat, scale, shift, win, 1e-3, W, b)
    plan = R.Plan(pos, scale, shift, lat.shape[1])
    p = pos.double().requires_grad_(True)
    h = R.encode_st(p, lat.double(), plan, win, 1e-3)
    for l in range(4):
        h = torch.nn.functional.linear(h, W[l].double(), b[l].double())
        if l < 3:
            h = torch.nn.functional.gelu(h)
    gx = torch.autograd.grad(h[:, 0].sum(), p)[0]
    assert rel(ref["sdf"], h[:, 0].detach()) < 1e-12
    assert ref["grad"].shape == (200, 4)
    assert rel(ref["grad"][:, :3], gx[:, :3]) < 1e-12 and rel(ref["grad"][:, 3], gx[:, 3]) < 1e-12
