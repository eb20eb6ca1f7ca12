"""Sphere-fit phase (Trainer.fit_sphere, DirectIteration.sphere_fit, psdf_sphere_fit_loss): the loss kernel against fp64 torch, one fit
iteration of the direct sequence against the autograd formulation, the optimizer semantics of the phase (SDF group only), graph replay
against eager, and the training step that follows the fit."""
import numpy as np
import pytest
import torch

import scenes

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _fresh_rngs():
    from permuto_sdf import OccupancyGrid, RaySampler, RaySamplesPacked, VolumeRendering
    from permuto_sdf_b200.permuto_sdf import _Pcg32Host
    OccupancyGrid.m_rng, RaySampler.m_rng, VolumeRendering.m_rng = _Pcg32Host(), _Pcg32Host(), _Pcg32Host()
    RaySamplesPacked.static_capacity = False


def _trainer(seed=5, **kw):
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.max_nr_samples_per_ray = 32
    hp.nr_samples_imp_sampling = 8
    hp.min_dist_between_samples = 1e-3
    kw.setdefault("optimizer", "fused")
    tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=128, nr_images=4, seed=seed, **kw)
    tr.set_analytic_scene()
    return tr


def _u01(n=30000, seed=7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(3, n, device="cuda", generator=g)


def _sdf_blocks(tr):
    """lattice, W_l, b_l gradients of the SDF model"""
    fs = tr.model_sdf.fused
    out = {"lattice": tr.model_sdf.encoding.lattice_values.grad.clone()}
    for l, lin in enumerate(fs.lin):
        out["W%d" % l], out["b%d" % l] = lin.weight.grad.clone(), lin.bias.grad.clone()
    return out


def _group(opt, name, buf):
    g = next(g for g in opt.param_groups if g["name"] == name)
    return buf[g["_off"]:g["_off"] + g["_n"]].clone()


# ------------------------------------------------------------------------------------------------ 1. the loss kernel
@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("N", [1, 1000, 30000, 30001])
def test_sphere_fit_loss_kernel_against_fp64(cuda, N, deterministic):
    """loss and terms within 1e-5 relative (+ the fixed-point rounding in deterministic mode); every seed within 1e-5 of the largest seed
    of its tensor (rows where sdf is close to the
    target distance or |grad| close to 1 lose relative accuracy to the cancellation of fp32 inputs, in any formulation); a zero gradient
    row gives zero seeds; deterministic mode is bit-reproducible"""
    from permuto_sdf_b200 import call
    from permuto_sdf_b200.train import sdf_loss_sphere
    call("psdf_set_deterministic", 1 if deterministic else 0, 1, 1)
    try:
        g = torch.Generator(device="cuda").manual_seed(N)
        pos = (torch.rand(N, 3, device="cuda", generator=g) - 0.5) * 0.9
        sdf = (pos.norm(dim=-1) - 0.3) + 0.05 * torch.randn(N, device="cuda", generator=g)
        grad = torch.randn(N, 3, device="cuda", generator=g) * 0.8
        grad[N // 2] = 0.0                                   # zero gradient row
        center = [0.02, -0.01, 0.03]
        outs = []
        for _ in range(2):
            g_sdf, g_grad = torch.full((N,), float("nan"), device="cuda"), torch.full((N, 3), float("nan"), device="cuda")
            acc, loss, terms = torch.zeros(4, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(2, device="cuda")
            call("psdf_sphere_fit_loss", N, pos, sdf, grad, 0.3, center, 1.0, 3e3, 5e1, g_sdf, g_grad, acc, loss, terms)
            torch.cuda.synchronize()
            assert float(acc.abs().max()) == 0.0, "accumulators and ticket are left zero"
            outs.append((loss.clone(), terms.clone(), g_sdf.clone(), g_grad.clone()))
        p = pos.double()
        s = sdf.double().view(-1, 1).requires_grad_(True)
        gr = grad.double().requires_grad_(True)
        ref, ref_sdf, ref_eik = sdf_loss_sphere(p, s, gr, 0.3, center)
        ref.backward()
        loss, terms, g_sdf, g_grad = outs[0]
        # deterministic mode: every block sum is rounded to the 2^-34 fixed-point grid (half a step per block, then the mean over N)
        fx = (N + 255) // 256 * 2.0 ** -35 / N if deterministic else 0.0
        ref, ref_sdf, ref_eik = float(ref), float(ref_sdf), float(ref_eik)
        assert abs(float(loss) - ref) <= 1e-5 * abs(ref) + (3e3 + 5e1) * fx
        assert abs(float(terms[0]) - ref_sdf) <= 1e-5 * abs(ref_sdf) + fx
        assert abs(float(terms[1]) - ref_eik) <= 1e-5 * abs(ref_eik) + fx
        assert torch.isfinite(g_sdf).all() and torch.isfinite(g_grad).all()
        assert float(g_grad[N // 2].abs().max()) == 0.0
        rs, rg = s.grad.view(-1).cpu(), gr.grad.cpu()
        assert float((g_sdf.double().cpu() - rs).abs().max()) <= 1e-5 * float(rs.abs().max())
        assert float((g_grad.double().cpu() - rg).abs().max()) <= 1e-5 * float(rg.abs().max()) + 1e-30
        if deterministic:
            for a, b in zip(outs[0], outs[1]):
                assert torch.equal(a, b)
    finally:
        call("psdf_set_deterministic", 0, 0, 0)


# ------------------------------------------------------------------------------------------------ 2. one iteration, direct vs autograd
@pytest.mark.parametrize("it", [0, 2000, 3999])
def test_direct_fit_iteration_equals_autograd(cuda, it):
    from permuto_sdf_b200.train import loss_sphere_init
    _fresh_rngs()
    tr = _trainer()
    assert tr._direct is not None
    u01 = _u01()
    tr.fixed_random = {"sphere_fit_u01": u01}
    tr.optimizer.zero_grad(set_to_none=False)
    ref, _, _ = loss_sphere_init(30000, tr.aabb, tr.model_sdf, it, points=tr.aabb.rand_points_inside_u01(u01))
    ref.backward()
    torch.cuda.synchronize()
    want = _sdf_blocks(tr)
    rest = {g["name"]: _group(tr.optimizer, g["name"], tr.optimizer.flat_grad) for g in tr.optimizer.param_groups if g["name"] != "model_sdf"}
    tr.optimizer.flat_grad.zero_()
    loss = tr._direct.sphere_fit(it, 30000, 0.3, [0.0, 0.0, 0.0])
    torch.cuda.synchronize()
    got = _sdf_blocks(tr)
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)), (float(loss), float(ref))
    for k in want:
        assert float(want[k].abs().max()) > 0, k
        assert rel(got[k], want[k]) < 2e-4, (k, rel(got[k], want[k]))
    for name, g in rest.items():                         # neither formulation touches the other models
        assert float(g.abs().max()) == 0.0 and float(_group(tr.optimizer, name, tr.optimizer.flat_grad).abs().max()) == 0.0, name


# ------------------------------------------------------------------------------------------------ 3. optimizer semantics of the phase
def _reference_fit(tr, u01, iters):
    """the autograd loop: loss_sphere_init + backward + FusedAdamW.step over the SDF group"""
    from permuto_sdf_b200.train import loss_sphere_init
    gi = [i for i, g in enumerate(tr.optimizer.param_groups) if g["name"] == "model_sdf"]
    for i in range(iters):
        tr.optimizer.zero_grad(set_to_none=False)
        loss, _, _ = loss_sphere_init(30000, tr.aabb, tr.model_sdf, i, points=tr.aabb.rand_points_inside_u01(u01))
        loss.backward()
        tr.optimizer.step(groups=gi)
        tr.model_sdf.fused.repack()
    return loss.detach()


def test_fit_steps_only_the_sdf_group(cuda):
    _fresh_rngs()
    u01 = _u01()
    a, b = _trainer(deterministic=True), _trainer(deterministic=True)
    opt = a.optimizer
    others = [g["name"] for g in opt.param_groups if g["name"] != "model_sdf"]
    before = {n: [_group(opt, n, t) for t in (opt.flat_param, opt.exp_avg, opt.exp_avg_sq)] for n in others}
    a.fixed_random = {"sphere_fit_u01": u01}
    loss = a.fit_sphere(5)
    ref = _reference_fit(b, u01, 5)
    torch.cuda.synchronize()
    assert a.execution["sphere_fit"].startswith("direct kernel sequence")
    assert a.sphere_fit_iter == 5 and a.iter_nr == 0 and opt.step_count == 5 == b.optimizer.step_count
    assert abs(float(loss) - float(ref)) <= 1e-4 * abs(float(ref))
    pa, pb = _group(opt, "model_sdf", opt.flat_param), _group(b.optimizer, "model_sdf", b.optimizer.flat_param)
    assert float((pa - pb).abs().max()) <= 1e-4, float((pa - pb).abs().max())
    for n in others:
        for x, y in zip(before[n], [_group(opt, n, t) for t in (opt.flat_param, opt.exp_avg, opt.exp_avg_sq)]):
            assert torch.equal(x, y), n
    assert float(opt.flat_grad.abs().max()) == 0.0
    t = a.last["sphere_fit_terms"]
    assert abs(float(t[0]) * 3e3 + float(t[1]) * 5e1 - float(loss)) <= 1e-5 * float(loss)


def test_fit_with_torch_adamw_leaves_other_parameters_stateless(cuda):
    _fresh_rngs()
    tr = _trainer(optimizer="adamw")
    tr.fixed_random = {"sphere_fit_u01": _u01()}
    loss = tr.fit_sphere(2)
    assert tr.execution["sphere_fit"].startswith("torch.autograd") and np.isfinite(float(loss)) and tr.sphere_fit_iter == 2
    for g in tr.optimizer.param_groups:
        for p in g["params"]:
            st = tr.optimizer.state.get(p, {})
            assert (len(st) > 0) == (g["name"] == "model_sdf" and p.requires_grad), g["name"]


# ------------------------------------------------------------------------------------------------ 4. graph replay
def _fit_params(graph, splits):
    _fresh_rngs()
    tr = _trainer(deterministic=True)
    tr.fixed_random = {"sphere_fit_u01": _u01()}
    if graph:
        tr.enable_cuda_graph()
    losses = [float(tr.fit_sphere(k)) for k in splits]
    assert tr.execution["sphere_fit"].endswith("CUDA-graph replay") == graph
    captured = tr._fit["graph"] is not None
    p, m = tr.optimizer.flat_param.clone(), tr.optimizer.exp_avg_sq.clone()
    step = tr.optimizer.step_count
    tr.disable_cuda_graph()
    _fresh_rngs()
    return p, m, losses, step, captured


def test_graph_replay_equals_eager_fit(cuda):
    pe, me, le, se, _ = _fit_params(False, [10])
    pg, mg, lg, sg, captured = _fit_params(True, [10])
    pg2, mg2, lg2, _, _ = _fit_params(True, [3, 7])
    assert captured and se == sg == 10
    assert torch.equal(pe, pg) and torch.equal(me, mg) and le == lg
    assert torch.equal(pg, pg2) and torch.equal(mg, mg2) and lg2[-1] == lg[-1]


# ------------------------------------------------------------------------------------------------ 5. training after the fit
def _rays(n=256):
    from permuto_sdf import PermutoSDF

    class Reel:
        pass
    rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)
    reel = Reel()
    reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
    gen = torch.Generator().manual_seed(3)
    pix = torch.randint(0, 60 * 80, (n,), generator=gen, dtype=torch.int32).cuda()
    img = torch.randint(0, 4, (n,), generator=gen, dtype=torch.int32).cuda()
    with torch.no_grad():
        return PermutoSDF.rays_from_reel_indices(reel, pix, img)


def test_training_step_after_fit(cuda):
    o, d, gt, gm, img = _rays()
    u01 = _u01()
    fixed = {"sphere_fit_u01": u01}

    def draw(name, fn):
        # the iteration's torch-RNG draws (off-surface points, curvature directions): the first trainer draws them, the second reuses them
        if name not in fixed:
            fixed[name] = fn()
        return fixed[name]
    res = {}
    for direct_fit in (True, False):
        _fresh_rngs()
        tr = _trainer(deterministic=True)
        tr.draw = draw
        if direct_fit:
            tr.fit_sphere(5)
        else:
            _reference_fit(tr, u01, 5)
            tr.sphere_fit_iter = 5
        assert tr.iter_nr == 0 and tr.execution["iteration"].startswith("direct kernel sequence")
        loss = tr.step(o, d, gt, gm, img, optimizer_step=False)
        torch.cuda.synchronize()
        assert tr.iter_nr == 1
        res[direct_fit] = (float(loss), {g["name"]: _group(tr.optimizer, g["name"], tr.optimizer.flat_grad) for g in tr.optimizer.param_groups})
    (la, ga), (lb, gb) = res[True], res[False]
    assert abs(la - lb) <= 1e-5 * abs(lb), (la, lb)
    for name in gb:
        assert float(gb[name].abs().max()) > 0, name
        assert rel(ga[name], gb[name]) < 2e-4, (name, rel(ga[name], gb[name]))
