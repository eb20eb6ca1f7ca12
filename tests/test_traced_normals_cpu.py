"""Sphere tracing with a box boundary and at a time value, without a GPU: the refusals of the tracer's entry points (Python and C ABI),
filter_unconverged_points against the reference's formula (sdf_utils.py:221-231), and the internal consistency of the reference
fixture tests/golden/refpy_golden_trace.npz (make_trace_golden.py), including AABB.ray_intersection restated op by op in torch
(aabb.py:47-100), which tests/test_traced_normals_gpu.py also uses as the yardstick of the kernel."""
import os
import types

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refpy_golden_trace.npz")
CASES = ["d3", "d4_a", "d4_b"]


def aabb_ray_intersection_torch(sizes, translation, ray_origins, ray_dirs):
    """aabb.py:47-100 as torch ops on the device of the rays, one op per step of the reference: fp32 box bounds, IEEE division,
    torch.where selections, the miss value 0 and the clamp of t_entry at 0"""
    dev = ray_origins.device
    size = torch.tensor(sizes, dtype=torch.float32, device=dev)
    trans = torch.tensor(translation, dtype=torch.float32, device=dev)
    bb_min = -size / 2 + trans
    bb_max = size - size / 2 + trans
    lo = -torch.ones_like(ray_origins[:, 0:1]) * 1e10
    hi = torch.ones_like(ray_origins[:, 0:1]) * 1e10
    miss = torch.zeros_like(ray_origins[:, 0:1]).bool()
    for i in range(3):
        a = ((bb_min[i] - ray_origins[:, i]) / ray_dirs[:, i]).unsqueeze(-1)
        b = ((bb_max[i] - ray_origins[:, i]) / ray_dirs[:, i]).unsqueeze(-1)
        swap = a > b
        a, b = torch.where(swap, b, a), torch.where(swap, a, b)
        miss = torch.logical_or(miss, torch.logical_or(b < lo, a > hi))
        lo = torch.where(a > lo, a, lo)
        hi = torch.where(b < hi, b, hi)
    zero = torch.zeros(1, 1, device=dev)
    lo = torch.clamp(torch.where(miss, zero, lo), min=0.0)
    hi = torch.where(miss, zero, hi)
    return ray_origins + lo * ray_dirs, lo, ray_origins + hi * ray_dirs, hi, torch.logical_not(miss)


def same_bits(a, b):
    """equal values, NaN where the other is NaN"""
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.is_floating_point():
        na, nb = torch.isnan(a), torch.isnan(b)
        return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])
    return torch.equal(a, b)


def fixture():
    return dict(np.load(GOLDEN))


# ------------------------------------------------------------------------------------------------ refusals
def _fused_stub(pos_dim, boundary):
    return types.SimpleNamespace(pos_dim=pos_dim, model=types.SimpleNamespace(boundary_primitive=boundary))


def test_fused_tracer_refusals():
    from permuto_sdf_b200.fused import _fused_sdf_sphere_trace
    from permuto_sdf_b200.permuto_sdf import AABB
    box = AABB([1, 1, 1], [0, 0, 0])
    p = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="pos_dim 4"):
        _fused_sdf_sphere_trace(_fused_stub(4, box), p, p, 0, 10, 0.9, 1e-3)
    with pytest.raises(RuntimeError, match="time_val given for a pos_dim 3"):
        _fused_sdf_sphere_trace(_fused_stub(3, box), p, p, 0, 10, 0.9, 1e-3, time_val=0.5)
    with pytest.raises(RuntimeError, match="boundary_primitive is a str"):
        _fused_sdf_sphere_trace(_fused_stub(3, "box"), p, p, 0, 10, 0.9, 1e-3)
    with pytest.raises(RuntimeError, match="boundary_primitive is a NoneType"):
        _fused_sdf_sphere_trace(_fused_stub(4, None), p, p, 0, 10, 0.9, 1e-3, time_val=0.0)


def test_trace_boundary_values():
    """the sphere's radius and centre; the box's max_bounds (s / 2 in double, then fp32, as check_point_inside_primitive compares) and
    its translation"""
    from permuto_sdf_b200.fused import _trace_boundary
    from permuto_sdf_b200.permuto_sdf import AABB, Sphere
    box = AABB([0.3, 1.1, 0.7], [0.1, -0.2, 0.05])
    kind, b = _trace_boundary(types.SimpleNamespace(boundary_primitive=box))
    assert kind == 1 and b[:3] == [float(np.float32(s / 2)) for s in (0.3, 1.1, 0.7)] and b[3:] == [0.1, -0.2, 0.05]
    sph = Sphere.__new__(Sphere)
    sph.m_radius, sph.m_center = 0.5, [0.1, 0.2, 0.3]
    kind, b = _trace_boundary(types.SimpleNamespace(boundary_primitive=sph))
    assert kind == 0 and b == [0.5, 0.1, 0.2, 0.3, 0.0, 0.0]


def test_trace_normals_refusals():
    from permuto_sdf_b200.surface_fit import SpaceTimeFit, SurfaceFit
    stub = types.SimpleNamespace(points=torch.zeros(1, 3))
    with pytest.raises(RuntimeError, match="time value"):
        SpaceTimeFit.trace_normals(stub, torch.zeros(2, 3), torch.zeros(2, 3), None)
    with pytest.raises(RuntimeError, match=r"ray_origins must be a float32 tensor of shape \[N,3\]"):
        SurfaceFit._trace_normals(stub, torch.zeros(2, 4), torch.zeros(2, 3), None, 20, 0.9, 2e-4, None)
    with pytest.raises(RuntimeError, match="ray_dirs must be a float32"):
        SurfaceFit._trace_normals(stub, torch.zeros(2, 3), torch.zeros(2, 3, dtype=torch.float64), None, 20, 0.9, 2e-4, None)
    with pytest.raises(RuntimeError, match="2 ray origins but 3 directions"):
        SurfaceFit._trace_normals(stub, torch.zeros(2, 3), torch.zeros(3, 3), None, 20, 0.9, 2e-4, None)


def test_c_entry_refuses_before_any_launch():
    """psdf_sdf_sphere_trace_dim returns PSDF_ERR_UNSUPPORTED (-3) for another pos_dim or boundary kind before it touches the device"""
    import ctypes
    from permuto_sdf_b200._lib import load_library
    lib = load_library()
    b6, t3 = (ctypes.c_float * 6)(1, 0, 0, 0, 0, 0), (ctypes.c_float * 3)(0, 0, 0)
    for pos_dim, kind in ((2, 0), (5, 1), (3, 2), (4, -1)):
        rc = lib.psdf_sdf_sphere_trace_dim(pos_dim, 0.0, kind, b6, 1, 24, 2 ** 18, None, None, None, None, None, None, 1e-3, 32, 1, None,
                                           20, 0.9, 2e-4, None, 1, 1.0, t3, None, None, None, None)
        assert rc == -3, (pos_dim, kind, rc)


# ------------------------------------------------------------------------------------------------ filter_unconverged_points
def test_filter_unconverged_points_is_the_reference_formula():
    """a SIGNED comparison sdf < tresh (points far inside pass too), default threshold 0.01, gradients may be None"""
    from permuto_sdf_b200.train import filter_unconverged_points
    g = torch.Generator().manual_seed(3)
    pts, grad = torch.randn(1000, 3, generator=g), torch.randn(1000, 3, generator=g)
    sdf = torch.cat([torch.randn(990, 1, generator=g) * 0.02, torch.tensor([[0.01], [-0.5], [0.00999], [0.0100001], [-0.0], [0.0],
                                                                          [float("inf")], [-float("inf")], [1e-3], [-1e-3]])])
    for tresh in (None, 2e-4, 0.05):
        kw = {} if tresh is None else {"sdf_converged_tresh": tresh}
        t = 0.01 if tresh is None else tresh
        c = (sdf < t) * 1.0
        p, gr, ic = filter_unconverged_points(pts, sdf, grad, **kw)
        assert ic.dtype == torch.float32 and ic.shape == (1000, 1)
        assert same_bits(ic, c) and same_bits(p, pts * c) and same_bits(gr, grad * c)
        p2, gr2, ic2 = filter_unconverged_points(pts, sdf, None, **kw)
        assert gr2 is None and same_bits(p2, p) and same_bits(ic2, ic)
    assert float(filter_unconverged_points(pts, sdf, grad)[2][991]) == 1.0      # sdf -0.5: far inside, kept by the signed test


# ------------------------------------------------------------------------------------------------ the fixture
def test_fixture_is_consistent():
    G = fixture()
    for c in CASES:
        key = c[:2]
        o, d = torch.from_numpy(G[c + ".origins"]), torch.from_numpy(G[c + ".dirs"])
        n = o.shape[0]
        # the reference's ray_intersection outputs are reproduced by the torch restatement, bit for bit
        got = aabb_ray_intersection_torch(G[key + ".box_size"].tolist(), G[key + ".box_translation"].tolist(), o, d)
        for name, g in zip(("pts_entry", "t_entry", "pts_exit", "t_exit", "hit"), got):
            assert same_bits(g, torch.from_numpy(G[c + "." + name])), (c, name)
        te, tx, hit = (torch.from_numpy(G[c + "." + k]) for k in ("t_entry", "t_exit", "hit"))
        assert hit.dtype == torch.bool and bool((te >= 0).all())
        assert bool((te[~hit] == 0).all()) and bool((tx[~hit] == 0).all())
        # the edge cases the fixture is meant to hold
        assert int((~hit).sum()) > 10 and int((d == 0).sum()) > 50
        size, trans = torch.tensor(G[key + ".box_size"]).float(), torch.tensor(G[key + ".box_translation"]).float()
        assert int(((o - trans).abs() < size / 2).all(1).sum()) > 0.1 * n                        # origins inside the box
        assert int(((o == -size / 2 + trans) | (o == size - size / 2 + trans)).any(1).sum()) > 0  # origins on a face
        assert len(set(size.tolist())) == 3 and bool((trans != 0).all())                          # non-cubic and translated
        # the traced points and filter_unconverged_points
        end, sdf, grad, ic = (torch.from_numpy(G[c + "." + k]) for k in ("ray_end", "sdf", "grad", "is_converged"))
        assert end.shape == (n, 3) and sdf.shape == (n, 1) and grad.shape == (n, 3) and ic.shape == (n, 1)
        assert bool(torch.isfinite(end).all()) and bool(torch.isfinite(sdf).all())
        assert same_bits(ic, (sdf < 0.01) * 1.0)
        conv = float((sdf.abs() < float(G[c + ".tresh"])).float().mean())
        assert 0.1 < conv < 0.9 and 0.1 < float(ic.mean()) < 0.95, (c, conv, float(ic.mean()))   # a fair share converges
        assert (float(G[c + ".time_val"]) < 0) == (c == "d3")
    assert G["d4_a.time_val"] != G["d4_b.time_val"]
    assert os.path.getsize(GOLDEN) < 1 << 20
