"""SDF from an oriented point cloud (SurfaceFit, psdf_surface_fit_points, psdf_surface_fit_loss): the points kernel against index_select
and the reference's box formula, the loss kernel against fp64 torch autograd of sdf_loss, one direct iteration and five iterations against
the autograd formulations, graph replay against eager across the end of the coarse-to-fine ramp, convergence on analytic clouds, and the
checkpoint round trip."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _reduction_mode_off_after(cuda):
    """SurfaceFit(deterministic=True) switches the device's mode on; later tests start from the default"""
    yield
    from permuto_sdf_b200 import call
    call("psdf_set_deterministic", 0, 0, 0)


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def sphere_cloud(n, center=(0.1, -0.05, 0.08), radius=0.3, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = F.normalize(torch.randn(n, 3, device="cuda", generator=g), dim=-1)
    c = torch.tensor(center, device="cuda")
    return (c + radius * d).contiguous(), d.contiguous()


def sphere_sdf(p, center=(0.1, -0.05, 0.08), radius=0.3):
    return (p - torch.tensor(center, device=p.device)).norm(dim=-1) - radius


def torus_cloud(n, R=0.25, r=0.1, seed=0):
    """uniform on the torus surface: angle v accepted with probability (R + r cos v) / (R + r)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    us, vs, have = [], [], 0
    while have < n:
        u = torch.rand(2 * n, device="cuda", generator=g) * 2 * math.pi
        v = torch.rand(2 * n, device="cuda", generator=g) * 2 * math.pi
        keep = torch.rand(2 * n, device="cuda", generator=g) < (R + r * torch.cos(v)) / (R + r)
        us.append(u[keep]); vs.append(v[keep]); have += int(keep.sum())
    u, v = torch.cat(us)[:n], torch.cat(vs)[:n]
    nrm = torch.stack([torch.cos(v) * torch.cos(u), torch.cos(v) * torch.sin(u), torch.sin(v)], -1)
    pts = torch.stack([(R + r * torch.cos(v)) * torch.cos(u), (R + r * torch.cos(v)) * torch.sin(u), r * torch.sin(v)], -1)
    return pts.contiguous(), nrm.contiguous()


def torus_sdf(p, R=0.25, r=0.1):
    q = torch.stack([p[:, :2].norm(dim=-1) - R, p[:, 2]], -1)
    return q.norm(dim=-1) - r


def draws(P, Ns, No, seed=11):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {"surface_fit_idx": torch.randint(P, (Ns,), device="cuda", generator=g),
            "surface_fit_u01": torch.rand(No, 3, device="cuda", generator=g)}


def blocks(fit):
    fs = fit.model_sdf.fused
    out = {"lattice": fit.model_sdf.encoding.lattice_values.grad.clone()}
    for l, lin in enumerate(fs.lin):
        out["W%d" % l], out["b%d" % l] = lin.weight.grad.clone(), lin.bias.grad.clone()
    return out


def params(fit):
    fs = fit.model_sdf.fused
    out = {"lattice": fit.model_sdf.encoding.lattice_values.detach().clone()}
    for l, lin in enumerate(fs.lin):
        out["W%d" % l], out["b%d" % l] = lin.weight.detach().clone(), lin.bias.detach().clone()
    return out


# ------------------------------------------------------------------------------------------------ 1. points kernel
@pytest.mark.parametrize("P", [1, 100000])
@pytest.mark.parametrize("Ns, No", [(1, 1), (3000, 30000), (3001, 29999)])
def test_points_kernel_is_index_select_and_the_box_formula(cuda, P, Ns, No):
    from permuto_sdf_b200 import AABB, call
    g = torch.Generator(device="cuda").manual_seed(P + Ns)
    pts, nrm = torch.randn(P, 3, device="cuda", generator=g), torch.randn(P, 3, device="cuda", generator=g)
    d = draws(P, Ns, No, seed=Ns)
    idx, u01 = d["surface_fit_idx"], d["surface_fit_u01"]
    for size, trans in (([1.0, 1.0, 1.0], [0.0, 0.0, 0.0]), ([0.7, 1.3, 2.1], [0.05, -0.3, 0.123])):
        x, n = torch.full((Ns + No, 3), float("nan"), device="cuda"), torch.full((Ns, 3), float("nan"), device="cuda")
        call("psdf_surface_fit_points", P, Ns, No, pts, nrm, idx, u01, size, trans, x, n)
        s = torch.as_tensor(size, device="cuda")
        box = u01 * s - s / 2 + torch.as_tensor(trans, device="cuda")        # AABB.rand_points_inside (aabb.py:110-114)
        assert torch.equal(x[:Ns], torch.index_select(pts, 0, idx)) and torch.equal(n, torch.index_select(nrm, 0, idx))
        assert torch.equal(x[Ns:], box)
        assert torch.equal(AABB(size, trans).rand_points_inside_u01(u01), box)


def test_aabb_points_are_inside(cuda):
    from permuto_sdf_b200 import AABB
    box = AABB([0.6, 1.0, 0.4], [0.1, 0.2, -0.1])
    p = box.rand_points_inside(20000)
    assert p.shape == (20000, 3) and bool(box.check_point_inside_primitive(p).all())


# ------------------------------------------------------------------------------------------------ 2. loss kernel
def _loss_inputs(Ns, No, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    N = Ns + No
    sdf = torch.randn(N, device="cuda", generator=g) * 0.03
    grad = torch.randn(N, 3, device="cuda", generator=g) * 0.7
    nrm = F.normalize(torch.randn(Ns, 3, device="cuda", generator=g), dim=-1) * 1.3
    special = {"zero_sdf": [0, Ns], "zero_grad": [0], "unit_grad": [Ns]}
    sdf[0], sdf[Ns] = 0.0, 0.0                               # |sdf| and exp(-100 |sdf|) at zero
    grad[0] = 0.0                                            # ‖g‖ = 0 on a surface row
    grad[Ns] = torch.tensor([0.0, 0.0, -1.0])                # ‖g‖ = 1 on a box row
    if Ns > 1:
        grad[1] = torch.tensor([0.0, 1.0, 0.0])              # ‖g‖ = 1 on a surface row
        special["unit_grad"].append(1)
    if No > 1:
        grad[Ns + 1] = 0.0                                   # ‖g‖ = 0 on a box row
        special["zero_grad"].append(Ns + 1)
    return sdf, grad, nrm, special


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("Ns, No", [(1, 1), (3000, 30000), (3001, 29999), (1000, 1)])
def test_loss_kernel_against_fp64_autograd(cuda, Ns, No, deterministic):
    from permuto_sdf_b200 import call
    from permuto_sdf_b200.surface_fit import LOSS_SCALE, SDF_LOSS_WEIGHTS, sdf_loss
    call("psdf_set_deterministic", 1 if deterministic else 0, 1, 1)
    try:
        sdf, grad, nrm, special = _loss_inputs(Ns, No, Ns * 7 + No)
        N = Ns + No
        outs = []
        for _ in range(2):
            g_sdf, g_grad = torch.full((N,), float("nan"), device="cuda"), torch.full((N, 3), float("nan"), device="cuda")
            acc, loss, terms = torch.zeros(5, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(4, device="cuda")
            call("psdf_surface_fit_loss", Ns, No, sdf, grad, nrm, *SDF_LOSS_WEIGHTS, LOSS_SCALE, g_sdf, g_grad, acc, loss, terms)
            torch.cuda.synchronize()
            assert float(acc.abs().max()) == 0.0, "accumulators and ticket are left zero"
            outs.append((loss.clone(), terms.clone(), g_sdf.clone(), g_grad.clone()))
        s = sdf.double().view(-1, 1).requires_grad_(True)
        gr = grad.double().requires_grad_(True)
        ref = sdf_loss(s[:Ns], gr[:Ns], s[Ns:], gr[Ns:], nrm.double()) / 30000
        ref_terms = [float(t) for t in sdf_loss.terms]
        ref.backward()
        loss, terms, g_sdf, g_grad = outs[0]
        # deterministic mode: each block sum is rounded to the 2^-34 fixed-point grid (half a step per block), then divided by the count
        half = (N + 255) // 256 * 2.0 ** -35 if deterministic else 0.0
        fx = [half / N, half / Ns, half / Ns, half / No]
        assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)) + LOSS_SCALE * sum(w * f for w, f in zip(SDF_LOSS_WEIGHTS, fx))
        for q in range(4):
            assert abs(float(terms[q]) - ref_terms[q]) <= 1e-5 * abs(ref_terms[q]) + fx[q], (q, float(terms[q]), ref_terms[q])
        assert torch.isfinite(g_sdf).all() and torch.isfinite(g_grad).all()
        rs, rg = s.grad.view(-1), gr.grad
        # special rows: torch's seeds. Zero seeds are zero; the ‖g‖ = 0 surface row gets -(w_nrm scale / Ns) n̂ / 1e-8
        for i in special["zero_sdf"]:
            assert float(g_sdf[i]) == 0.0 == float(rs[i])
        for i in special["zero_grad"] + special["unit_grad"]:
            if i >= Ns:
                assert float(g_grad[i].abs().max()) == 0.0 == float(rg[i].abs().max())
            else:
                assert float((g_grad[i].double() - rg[i]).abs().max()) <= 1e-6 * float(rg[i].abs().max()), (i, g_grad[i], rg[i])
        want0 = -(SDF_LOSS_WEIGHTS[1] * LOSS_SCALE / Ns) * F.normalize(nrm[0].double(), dim=0) / 1e-8
        assert float((rg[0] - want0).abs().max()) <= 1e-9 * float(want0.abs().max())
        # every other row: within 1e-5 of the largest seed of its tensor
        keep = torch.ones(N, dtype=torch.bool, device="cuda")
        keep[special["zero_grad"] + special["unit_grad"]] = False
        if keep.any():
            assert float((g_sdf.double() - rs).abs().max()) <= 1e-5 * float(rs.abs().max())
            assert float((g_grad.double() - rg)[keep].abs().max()) <= 1e-5 * float(rg[keep].abs().max()) + 1e-30
        if deterministic:
            for a, b in zip(outs[0], outs[1]):
                assert torch.equal(a, b)
    finally:
        call("psdf_set_deterministic", 0, 0, 0)


def test_loss_kernel_refuses_empty_sets(cuda):
    from permuto_sdf_b200 import call
    z = lambda *s: torch.zeros(*s, device="cuda")
    for ns, no in ((0, 5), (5, 0)):
        with pytest.raises(RuntimeError, match="psdf_surface_fit_loss failed"):
            call("psdf_surface_fit_loss", ns, no, z(5), z(5, 3), z(5, 3), 1.0, 1.0, 1.0, 1.0, 1.0, z(5), z(5, 3), z(5), z(1), z(4))


# ------------------------------------------------------------------------------------------------ 3. one iteration, direct vs autograd
@pytest.mark.parametrize("it", [0, 2500, 5000])
@pytest.mark.parametrize("L, hidden", [(16, 32), (16, 64), (24, 32), (24, 64)])
def test_direct_iteration_equals_autograd(cuda, it, L, hidden):
    from permuto_sdf_b200 import SurfaceFit
    pts, nrm = sphere_cloud(50000)
    d = draws(50000, 3000, 30000)
    fits = {}
    for name, kw in (("direct", {}), ("fused", {"direct": False}), ("per_op", {"fused_training": False})):
        f = SurfaceFit(pts, nrm, nr_levels=L, hidden=hidden, seed=4, **kw)
        f.fixed_random = d
        fits[name] = f
    assert fits["direct"].direct and not fits["fused"].direct and not fits["per_op"].direct
    assert fits["per_op"].execution["step"].startswith("torch.autograd")
    p0 = params(fits["direct"])
    for f in fits.values():
        assert all(torch.equal(p0[k], v) for k, v in params(f).items())
    loss = fits["direct"]._direct_forward_backward(it, 3000, 30000)
    ref = fits["fused"]._autograd_forward_backward(it, 3000, 30000)
    ref2 = fits["per_op"]._autograd_forward_backward(it, 3000, 30000)
    torch.cuda.synchronize()
    got, want, want2 = blocks(fits["direct"]), blocks(fits["fused"]), blocks(fits["per_op"])
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)), (float(loss), float(ref))
    assert abs(float(loss) - float(ref2)) <= 1e-4 * abs(float(ref2)), (float(loss), float(ref2))
    assert rel(fits["direct"].last["terms"], fits["fused"].last["terms"]) < 1e-5
    for k in want:
        assert float(want[k].abs().max()) > 0, k
        assert rel(got[k], want[k]) < 2e-4, (k, rel(got[k], want[k]))
        assert rel(got[k], want2[k]) < 1e-3, (k, rel(got[k], want2[k]))


# ------------------------------------------------------------------------------------------------ 4. five iterations
def test_five_iterations_against_the_torch_adamw_loop(cuda):
    from permuto_sdf_b200 import SurfaceFit
    pts, nrm = torus_cloud(50000)
    d = draws(50000, 3000, 30000, seed=3)
    a = SurfaceFit(pts, nrm, seed=2, deterministic=True)
    b = SurfaceFit(pts, nrm, seed=2, optimizer="adamw", deterministic=True)
    assert a.execution["step"].startswith("direct kernel sequence") and b.execution["step"].startswith("torch.autograd")
    a.fixed_random, b.fixed_random = d, d
    la = a.fit(5)
    lb = None
    for _ in range(5):
        lb = b.step()
    torch.cuda.synchronize()
    assert a.iter_nr == b.iter_nr == 5 and a.optimizer.step_count == 5
    assert abs(float(la) - float(lb)) <= 1e-4 * abs(float(lb)), (float(la), float(lb))
    pa, pb = params(a), params(b)
    for k in pa:
        assert rel(pa[k], pb[k]) < 2e-4, (k, rel(pa[k], pb[k]))
    assert float(a.optimizer.flat_grad.abs().max()) == 0.0
    t = a.last["terms"]
    w = (5e1, 1e2, 3e3, 1e2)
    assert abs(sum(float(t[q]) * w[q] for q in range(4)) / 30000 - float(la)) <= 1e-5 * float(la)


# ------------------------------------------------------------------------------------------------ 5. graph replay
def _run(graph, splits, c2f=6):
    from permuto_sdf_b200 import SurfaceFit
    pts, nrm = sphere_cloud(20000)
    f = SurfaceFit(pts, nrm, nr_levels=16, capacity=2 ** 14, nr_iters_for_c2f=c2f, deterministic=True, seed=9)
    f.fixed_random = draws(20000, 1000, 5000, seed=5)
    if graph:
        f.enable_cuda_graph()
    losses = [float(f.fit(k, 1000, 5000)) for k in splits]
    assert f.execution["step"].endswith("CUDA-graph replay") == graph
    captures = f._cg["captures"] if graph else 0
    out = (f.optimizer.flat_param.clone(), f.optimizer.exp_avg_sq.clone(), losses, f.iter_nr, captures)
    f.disable_cuda_graph()
    return out


def test_graph_replay_equals_eager_across_the_window_ramp(cuda):
    pe, me, le, ie, _ = _run(False, [10])
    pg, mg, lg, ig, cap = _run(True, [10])
    pg2, mg2, lg2, _, cap2 = _run(True, [4, 6])
    assert ie == ig == 10
    assert cap == 2 and cap2 == 2, (cap, cap2)         # iterations [1, 6) on the ramp, then [6, ...) with the open window
    assert torch.equal(pe, pg) and torch.equal(me, mg) and le == lg
    assert torch.equal(pg, pg2) and torch.equal(mg, mg2) and lg2[-1] == lg[-1]


# ------------------------------------------------------------------------------------------------ 6. convergence
@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_convergence_on_analytic_clouds(cuda, shape):
    from permuto_sdf_b200 import SurfaceFit
    cloud, true_sdf = (sphere_cloud, sphere_sdf) if shape == "sphere" else (torus_cloud, torus_sdf)
    pts, nrm = cloud(200000, seed=1)
    f = SurfaceFit(pts, nrm)
    f.enable_cuda_graph()
    f.fit(3000)
    torch.cuda.synchronize()
    hp, hn = cloud(10000, seed=2)
    with torch.no_grad():
        sdf, grad, _ = f.model_sdf.fused(hp, f.iter_nr, with_gradient=True, with_geom=False)
        mean_abs = float(sdf.abs().mean())
        mean_cos = float((1 - F.cosine_similarity(grad, hn, dim=-1)).mean())
        g = torch.Generator(device="cuda").manual_seed(3)
        box = torch.rand(200000, 3, device="cuda", generator=g) - 0.5
        ts = true_sdf(box)
        far = ts.abs() > 0.05
        s_box, _, _ = f.model_sdf.fused(box[far], f.iter_nr, with_gradient=False, with_geom=False)
        sign_ok = float(((s_box.view(-1) > 0) == (ts[far] > 0)).float().mean())
    print("surface fit %s: mean |sdf| %.3e, mean 1 - cos %.3e, sign correct %.5f, loss %.4e" % (
        shape, mean_abs, mean_cos, sign_ok, float(f.last["terms"][0])))
    assert mean_abs < 2e-3 and mean_cos < 1e-2 and sign_ok >= 0.99, (mean_abs, mean_cos, sign_ok)


# ------------------------------------------------------------------------------------------------ 7. checkpoints
def test_save_load_resumes_bit_for_bit(cuda, tmp_path):
    import refshape_models as R
    from permuto_sdf_b200 import SurfaceFit
    pts, nrm = sphere_cloud(20000)
    d = draws(20000, 1000, 5000, seed=8)
    mk = lambda: SurfaceFit(pts, nrm, nr_levels=16, capacity=2 ** 14, deterministic=True, seed=6)
    a = mk()
    a.fixed_random = d
    a.fit(3, 1000, 5000)
    path = a.save(str(tmp_path), "sdf_from_mesh")
    a.fit(3, 1000, 5000)
    b = mk()
    b.fixed_random = d
    b.load(path)
    assert b.iter_nr == 3 and b.optimizer.step_count == 3
    b.fit(3, 1000, 5000)
    assert torch.equal(a.optimizer.flat_param, b.optimizer.flat_param) and torch.equal(a.optimizer.exp_avg, b.optimizer.exp_avg)
    # sdf_model.pt is the reference model's state_dict: the reference-shaped SDF reads it strictly
    sd = torch.load(path + "/sdf_model.pt")
    ref = R.SDF(3, None, 0, 5000, nr_levels=16, capacity=2 ** 14)
    assert sorted(sd) == sorted(ref.state_dict())
    ref.load_state_dict(sd)
    # a checkpoint of the reference (no optimizer state) loads with iter_nr = 0
    import os
    os.remove(path + "/surface_fit_state.pt")
    c = mk()
    c.iter_nr = 17
    c.load(path)
    assert c.iter_nr == 0 and torch.equal(c.model_sdf.encoding.lattice_values, sd["encoding.lattice_values"])
