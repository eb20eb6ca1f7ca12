"""Sphere tracing with a box boundary and at a time value on the GPU: psdf_aabb_ray_intersection bit for bit against aabb.py restated in
torch and against the reference fixture; the fused tracer (k_sdf_sphere_trace<D, BOX>) bit for bit against the masked gather / scatter
loop on the same network at D = 3 / 4, sphere / box boundary, with and without an occupancy grid; the original entry point against the
new one; SurfaceFit.trace_normals and SpaceTimeFit.trace_normals against the reference's own sphere_trace (make_trace_golden.py), their
freedom from side effects, and traced points on the analytic surface after the existing convergence runs."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_fused_backward_fp64_gpu import sms
from test_fused_forward_fp64_gpu import SENTINEL
from test_surface_fit_gpu import sphere_cloud, sphere_sdf
from test_spacetime_fit_gpu import moving_sphere, sequence
from test_traced_normals_cpu import CASES, aabb_ray_intersection_torch, fixture, same_bits

pytestmark = pytest.mark.gpu
GUARD = 8


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rays_at_box(n, size, trans, seed, axis_share=0.1):
    """rays towards points of the box from outside, away from it, from inside, and with direction components exactly 0"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    size, trans = torch.tensor(size, device="cuda"), torch.tensor(trans, device="cuda")
    o = trans + F.normalize(torch.randn(n, 3, device="cuda", generator=g), dim=-1) * (0.3 + 1.5 * torch.rand(n, 1, device="cuda", generator=g))
    target = trans + (torch.rand(n, 3, device="cuda", generator=g) - 0.5) * size
    d = target - o
    away = torch.rand(n, device="cuda", generator=g) < 0.15
    d[away] = -d[away]
    axis = torch.rand(n, device="cuda", generator=g) < axis_share
    k = torch.randint(3, (n,), device="cuda", generator=g)
    d[axis, k[axis]] = 0.0
    return o.contiguous(), F.normalize(d, dim=-1).contiguous()


# ------------------------------------------------------------------------------------------------ AABB.ray_intersection
def test_aabb_ray_intersection_matches_torch_formula(cuda):
    from permuto_sdf_b200.permuto_sdf import AABB
    boxes = [([1.0, 1.0, 1.0], [0.0, 0.0, 0.0]), ([0.9, 1.1, 0.8], [0.05, -0.1, 0.02]), ([0.3, 2.0, 0.7], [-0.4, 0.25, 0.1])]
    for bi, (size, trans) in enumerate(boxes):
        o, d = rays_at_box(1 << 20, size, trans, seed=bi, axis_share=0.2)
        # edge cases: axis-parallel rays, origins on the faces (0 / 0), zero direction, origins at the corners, rays along a face
        s, t = torch.tensor(size, device="cuda"), torch.tensor(trans, device="cuda")
        bmin, bmax = -s / 2 + t, s - s / 2 + t
        eo = torch.stack([bmin, bmax, (bmin + bmax) / 2, bmin * 3, torch.stack([bmin[0], bmax[1], t[2]]), torch.zeros(3, device="cuda")])
        ed = torch.eye(3, device="cuda")
        ed = torch.cat([ed, -ed, torch.zeros(1, 3, device="cuda"), F.normalize(torch.ones(1, 3, device="cuda"), dim=-1)])
        o = torch.cat([o, eo.repeat_interleave(ed.shape[0], 0)]).contiguous()
        d = torch.cat([d, ed.repeat(eo.shape[0], 1)]).contiguous()
        got = AABB(size, trans).ray_intersection(o, d)
        want = aabb_ray_intersection_torch(size, trans, o, d)
        for name, a, b in zip(("pts_entry", "t_entry", "pts_exit", "t_exit", "hit"), got, want):
            assert a.shape == b.shape and same_bits(a, b), (bi, name)
        assert int((~got[4]).sum()) > 1000 and bool(torch.isnan((bmin[0] - o[:, 0]) / d[:, 0]).any())      # misses and 0 / 0


@pytest.mark.parametrize("case", CASES)
def test_aabb_ray_intersection_matches_fixture(cuda, case):
    from permuto_sdf_b200.permuto_sdf import AABB
    G = fixture()
    key = case[:2]
    got = AABB(G[key + ".box_size"].tolist(), G[key + ".box_translation"].tolist()).ray_intersection(cu(G[case + ".origins"]),
                                                                                                    cu(G[case + ".dirs"]))
    for name, a in zip(("pts_entry", "t_entry", "pts_exit", "t_exit", "hit"), got):
        assert same_bits(a.cpu(), torch.from_numpy(G[case + "." + name])), name


# ------------------------------------------------------------------------------------------------ the tracer against the masked loop
def fixture_model(key):
    """the fixture's SDF (D = 3 or 4, its AABB) with the hash table regenerated from its seed, on the fused inference path"""
    from test_refpy_golden_gpu import lattice_from_seed
    from permuto_sdf_b200.models import SDF
    from permuto_sdf_b200.permuto_sdf import AABB
    G = fixture()
    D = 3 if key == "d3" else 4
    aabb = AABB(G[key + ".box_size"].tolist(), G[key + ".box_translation"].tolist())
    m = SDF(D, aabb, 0, 5000 if D == 3 else 3000).cuda()
    sd = {k[len(key + ".state."):]: torch.from_numpy(v) for k, v in G.items() if k.startswith(key + ".state.")}
    sd["encoding.lattice_values"] = lattice_from_seed(int(G[key + ".seed"]), 24, 2 ** 18, 2, 1.0) * torch.from_numpy(G[key + ".level_amp"]).view(-1, 1, 1)
    m.load_state_dict(sd, strict=True)
    m.enable_fused_inference()
    m.eval()
    m.last_iter_nr = int(G[key + ".iter"])
    return m, aabb


def occupancy(seed):
    from permuto_sdf_b200.permuto_sdf import OccupancyGrid
    grid = OccupancyGrid(64, 1.0, [0, 0, 0])
    g = torch.Generator(device="cuda").manual_seed(seed)
    grid.set_grid_occupancy((torch.rand(64 ** 3, device="cuda", generator=g) < 0.7).contiguous())
    return grid


@pytest.mark.parametrize("grid", [False, True], ids=["boundary", "grid"])
@pytest.mark.parametrize("boundary", ["sphere", "box"])
@pytest.mark.parametrize("D", [3, 4])
def test_fused_tracer_equals_masked_loop(cuda, D, boundary, grid):
    """train.sphere_trace on the fused tracer and on the masked loop give the same bits (points, final sdf, gradient); without a grid the
    tracer is also called directly on the loop's start points with NaN-sentinel guard rows past N, which it must not write"""
    import permuto_sdf_b200.train as tr
    from permuto_sdf_b200._lib import call
    from permuto_sdf_b200.fused import _trace_boundary
    from permuto_sdf_b200.permuto_sdf import Sphere
    m, aabb = fixture_model("d3" if D == 3 else "d4")
    if boundary == "sphere":
        m.boundary_primitive = Sphere(0.55, aabb.bounding_box_translation)
    occ = occupancy(D) if grid else None
    runs = [(n, 0.37) for n in (1, 127, 128, 2 * 128 * sms() + 5)] + ([(2 * 128 * sms() + 5, t) for t in (0.0, 1.0)] if D == 4 else [])
    for n, t in runs:
        time_val = t if D == 4 else None
        o, d = rays_at_box(n, aabb.bounding_box_sizes_xyz, aabb.bounding_box_translation, seed=n + D)
        res = {}
        for fused in (False, True):
            tr.FUSED_SPHERE_TRACE = fused
            try:
                with torch.no_grad():
                    pts, sdf, grads, _, _ = tr.sphere_trace(20, o, d, m, True, 0.9, 2e-4, occ, time_val)
            finally:
                tr.FUSED_SPHERE_TRACE = True
            res[fused] = (pts.clone(), sdf.clone(), grads.clone())
        assert all(torch.equal(a, b) for a, b in zip(res[True], res[False])), (n, t, float((res[True][0] - res[False][0]).abs().max()))
        assert bool(torch.isfinite(res[True][0]).all())
        if n > 1000:
            assert 0.02 < float((res[True][1].abs() < 2e-4).float().mean()) < 0.98       # a fair share of the rays converges
        if grid:
            continue
        pe = m.boundary_primitive.ray_intersection(o, d)[0]
        kind, b6 = _trace_boundary(m)
        enc, fs = m.encoding, m.fused
        out = torch.full((n + GUARD, 3), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
        conv = torch.full((n + GUARD,), 0xAB, dtype=torch.uint8, device="cuda")
        queue = torch.zeros(8, dtype=torch.int32, device="cuda")
        call("psdf_sdf_sphere_trace_dim", D, 0.0 if time_val is None else time_val, kind, b6, n, enc.nr_levels, enc.capacity, pe, d,
             enc.lattice_values.detach(), enc.scale_factor, enc.shift_tensor(), m.window(m.last_iter_nr).view(-1).contiguous(),
             enc.concat_points_scaling, fs.hidden, fs.out_dim, fs.blob, 20, 0.9, 2e-4, None, 1, 1.0, [0.0, 0.0, 0.0], out, conv, queue)
        assert torch.equal(out[:n], res[False][0])
        assert bool((out[n:].view(torch.int32) == SENTINEL).all()) and bool((conv[n:] == 0xAB).all()) and bool((conv[:n] <= 1).all())


def test_original_entry_point_equals_dim_3_sphere(cuda):
    """psdf_sdf_sphere_trace is the (3, sphere) case of psdf_sdf_sphere_trace_dim: the same bits, with and without an occupancy grid"""
    from permuto_sdf_b200._lib import call
    m, aabb = fixture_model("d3")
    enc, fs = m.encoding, m.fused
    n = 2 * 128 * sms() + 5
    o, d = rays_at_box(n, aabb.bounding_box_sizes_xyz, aabb.bounding_box_translation, seed=5)
    radius, center = 0.55, [0.05, -0.1, 0.02]
    net = lambda: (n, enc.nr_levels, enc.capacity, o, d, enc.lattice_values.detach(), enc.scale_factor, enc.shift_tensor(),
                   m.window(5000).view(-1).contiguous(), enc.concat_points_scaling, fs.hidden, fs.out_dim, fs.blob, 20, 0.9, 2e-4)
    for grid in (None, occupancy(9)):
        geo = (grid.m_grid_occupancy, *grid._geom()) if grid is not None else (None, 1, 1.0, [0.0, 0.0, 0.0])
        outs = []
        for dim in (False, True):
            out, conv, q = torch.empty(n, 3, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda"), torch.zeros(8, dtype=torch.int32, device="cuda")
            if dim:
                call("psdf_sdf_sphere_trace_dim", 3, 0.0, 0, [radius] + center + [0.0, 0.0], *net(), *geo, out, conv, q)
            else:
                call("psdf_sdf_sphere_trace", *net(), *geo, radius, center, out, conv, q)
            outs.append((out, conv))     # (the launch statistics in q depend on the order in which CTAs claim rays, not on the entry point)
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


# ------------------------------------------------------------------------------------------------ against the reference
def load_fit(key, G):
    """SurfaceFit / SpaceTimeFit with the fixture's box, state and hash table"""
    from test_refpy_golden_gpu import lattice_from_seed
    from permuto_sdf_b200 import SpaceTimeFit, SurfaceFit
    size, trans = G[key + ".box_size"].tolist(), G[key + ".box_translation"].tolist()
    if key == "d3":
        pts, nrm = sphere_cloud(1000)
        f = SurfaceFit(pts, nrm, box_size=size, box_translation=trans)
    else:
        pts, nrm = sequence(5)
        f = SpaceTimeFit(pts, nrm, box_size=size, box_translation=trans)
    sd = {k[len(key + ".state."):]: torch.from_numpy(v) for k, v in G.items() if k.startswith(key + ".state.")}
    sd["encoding.lattice_values"] = lattice_from_seed(int(G[key + ".seed"]), 24, 2 ** 18, 2, 1.0) * torch.from_numpy(G[key + ".level_amp"]).view(-1, 1, 1)
    f.model_sdf.load_state_dict(sd, strict=True)
    return f


@pytest.mark.parametrize("case", CASES)
def test_trace_normals_against_reference(cuda, case):
    """The tensor-core network and the CPU oracle agree to the existing bars (sdf 1e-4, gradient 1e-3), not bit for bit, so the traced
    points differ in their last bits and a ray's convergence can flip where a decision (|sdf| < 2e-4 at one of its <= 20 steps, or
    sdf < 0.01 in filter_unconverged_points) is taken on a value closer to the threshold than that disagreement. The field has
    |d sdf/dx| ~ 1 and the steps' sdf values are spread over ~1e-1, so a value falls within ~1e-5 of a threshold with probability ~1e-4
    per decision, ~2e-3 per ray over 20 steps; the bound on rays whose masks differ, 1 % of the rays plus 3, is several times that.
    Where both sides converged on the surface, sdf agrees to 1e-4; normals are compared at the same points (the reference's end points)
    to 1e-3: the end points themselves differ in their last bits, and on this hash-grid field the gradient changes abruptly across
    lattice cells, so the normal at a point 1e-6 away is not a measure of the evaluation. Rays that have not converged after the last
    step are still in flight and their end points are not compared."""
    G = fixture()
    key = case[:2]
    f = load_fit(key, G)
    o, d = cu(G[case + ".origins"]), cu(G[case + ".dirs"])
    it = int(G[key + ".iter"])
    mult, tresh, iters = float(G[case + ".mult"]), float(G[case + ".tresh"]), int(G[case + ".nr_iters"])
    time_val = None if key == "d3" else float(G[case + ".time_val"])
    if key == "d3":
        ray_end, normals, normals_conv, is_conv = f.trace_normals(o, d, iters, mult, tresh, iter_nr=it)
    else:
        ray_end, normals, normals_conv, is_conv = f.trace_normals(o, d, time_val, iters, mult, tresh, iter_nr=it)
    n = o.shape[0]
    assert ray_end.shape == (n, 3) and normals.shape == (n, 3) and normals_conv.shape == (n, 3) and is_conv.shape == (n, 1)
    ref_end, ref_sdf, ref_grad, ref_conv = (cu(G[case + "." + k]) for k in ("ray_end", "sdf", "grad", "is_converged"))
    ref_n = F.normalize(ref_grad, dim=1)
    fs = f.model_sdf.fused
    with_t = lambda p: (p if time_val is None else torch.cat([p, torch.full((n, 1), time_val, device="cuda")], 1)).contiguous()
    with torch.no_grad():
        sdf = fs(with_t(ray_end), it, with_gradient=False, with_geom=False)[0]          # the trace's final evaluation
        sdf_at_ref, grad_at_ref, _ = fs(with_t(ref_end), it, with_gradient=True, with_geom=False)
    on_surface = ((ref_sdf.abs() < tresh) & (sdf.abs() < tresh)).view(-1)
    flips = int(((ref_sdf.abs() < tresh) != (sdf.abs() < tresh)).sum()) + int((is_conv != ref_conv).sum())
    dn_ref = (F.normalize(grad_at_ref, dim=1) - ref_n).abs().max(dim=1).values
    print("%s: %d rays, %d on the surface on both sides, %d mask differences, max |d sdf| there %.2e, max |d normal| at the reference's "
          "points %.2e" % (case, n, int(on_surface.sum()), flips, float((sdf - ref_sdf).abs().view(-1)[on_surface].max()),
                          float(dn_ref[ref_conv.view(-1) > 0].max())))
    assert flips <= 0.01 * n + 3
    assert int(on_surface.sum()) > 0.1 * n
    assert float((sdf - ref_sdf).abs().view(-1)[on_surface].max()) <= 1e-4
    assert float((sdf_at_ref - ref_sdf).abs().max()) <= 1e-4
    assert float(dn_ref[ref_conv.view(-1) > 0].max()) <= 1e-3
    # the outputs' own relations
    assert torch.equal(is_conv, (sdf < 0.01) * 1.0)
    assert torch.allclose(normals_conv, normals * is_conv, atol=1e-6)
    assert bool((normals_conv[is_conv.view(-1) == 0] == 0).all())


# ------------------------------------------------------------------------------------------------ no side effects
@pytest.mark.parametrize("space_time", [False, True], ids=["SurfaceFit", "SpaceTimeFit"])
def test_trace_normals_has_no_side_effects(cuda, space_time):
    from permuto_sdf_b200 import SpaceTimeFit, SurfaceFit
    if space_time:
        pts, nrm = sequence(20)
        f = SpaceTimeFit(pts, nrm, nr_levels=16, capacity=2 ** 14, seed=2)
    else:
        pts, nrm = sphere_cloud(20000)
        f = SurfaceFit(pts, nrm, nr_levels=16, capacity=2 ** 14, seed=2)
    f.enable_cuda_graph()
    f.fit(4, 1000, 2000)
    torch.cuda.synchronize()
    opt, m = f.optimizer, f.model_sdf
    snap = lambda: ([p.detach().clone() for p in m.parameters()], [p.grad.clone() for p in m.parameters() if p.grad is not None],
                    [opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.flat_param.clone()], opt.step_count, f.iter_nr, m.training,
                    m.last_iter_nr, f._dev["it_dev"].clone(), f._dev["step_dev"].clone(), torch.cuda.get_rng_state(), torch.get_rng_state())
    before = snap()
    o, d = rays_at_box(5000, [1, 1, 1], [0, 0, 0], seed=4)
    out = f.trace_normals(o, d, 0.5) if space_time else f.trace_normals(o, d)
    torch.cuda.synchronize()
    after = snap()
    assert all(bool(torch.isfinite(t).all()) for t in out)
    for a, b in zip(before, after):
        if isinstance(a, list):
            assert all(torch.equal(x, y) for x, y in zip(a, b))
        elif isinstance(a, torch.Tensor):
            assert torch.equal(a, b)
        else:
            assert a == b
    f.fit(1, 1000, 2000)                          # training goes on from where it was
    assert f.iter_nr == 5


# ------------------------------------------------------------------------------------------------ end to end
def camera_rays(n_side, eye, look_at):
    """a pinhole camera's rays (n_side x n_side pixels, 40 degree field of view)"""
    eye, at = torch.tensor(eye, device="cuda"), torch.tensor(look_at, device="cuda")
    fwd = F.normalize(at - eye, dim=0)
    right = F.normalize(torch.linalg.cross(fwd, torch.tensor([0.0, 1.0, 0.0], device="cuda")), dim=0)
    up = torch.linalg.cross(right, fwd)
    s = (torch.arange(n_side, device="cuda").float() + 0.5) / n_side * 2 - 1
    v, u = torch.meshgrid(s, s, indexing="ij")
    tan = float(np.tan(np.radians(20)))
    d = F.normalize(fwd + tan * (u.reshape(-1, 1) * right + v.reshape(-1, 1) * up), dim=1)
    return eye.expand_as(d).contiguous(), d.contiguous()


def test_traced_points_lie_on_the_surface(cuda):
    """After the 3000-iteration runs of the existing convergence tests (SurfaceFit on the off-centre sphere, SpaceTimeFit on the moving
    sphere), the converged rays of a 200 x 200 camera end on the analytic surface: the median distance is below 2e-3 of the unit box,
    the bar of those tests for the mean |sdf| at surface points (the space-time one at a time between the frames)."""
    from permuto_sdf_b200 import SpaceTimeFit, SurfaceFit
    pts, nrm = sphere_cloud(200000, seed=1)
    f = SurfaceFit(pts, nrm)
    f.enable_cuda_graph()
    f.fit(3000)
    o, d = camera_rays(200, [0.1, 0.3, 1.4], [0.1, -0.05, 0.08])
    end, normals, _, _ = f.trace_normals(o, d)
    ok = (f.model_sdf.fused(end, f.iter_nr - 1, with_geom=False)[0].abs() < 2e-4).view(-1)
    dist = sphere_sdf(end[ok]).abs()
    print("surface fit: %d of %d rays converged, median distance %.2e" % (int(ok.sum()), ok.numel(), float(dist.median())))
    assert int(ok.sum()) > 0.15 * ok.numel() and float(dist.median()) < 2e-3
    pts, nrm = sequence(1000, seed=1)
    torch.manual_seed(123)
    f = SpaceTimeFit(pts, nrm)
    f.enable_cuda_graph()
    f.fit(3000)
    t = 0.4 + 0.5 / 220                           # between two frames of the sequence
    c, r = moving_sphere(torch.tensor([t], device="cuda"))
    o, d = camera_rays(200, [0.0, 0.3, 1.4], c.view(-1).tolist())
    end, normals, _, _ = f.trace_normals(o, d, t)
    with torch.no_grad():
        s = f.model_sdf.fused(torch.cat([end, torch.full((end.shape[0], 1), t, device="cuda")], 1).contiguous(), f.iter_nr - 1, with_geom=False)[0]
    ok = (s.abs() < 2e-4).view(-1)
    dist = ((end[ok] - c).norm(dim=1) - r).abs()
    print("space-time fit at t = %.4f: %d of %d rays converged, median distance %.2e" % (t, int(ok.sum()), ok.numel(), float(dist.median())))
    assert int(ok.sum()) > 0.08 * ok.numel() and float(dist.median()) < 2e-3
