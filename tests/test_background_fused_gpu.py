"""Fused background network (csrc/fused_bg.cu, fused.FusedNerfHash) against the reference's own NerfHash outputs and gradients
(tests/golden/refpy_golden_bg.npz) and against NerfHash on the per-op encoding kernels + autograd."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def rel(a, b):
    a = torch.as_tensor(a).detach().cpu().double().reshape(-1)
    b = torch.as_tensor(b).detach().cpu().double().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}


def test_fused_background_matches_reference_golden(cuda):
    """the fused kernels reproduce NerfHash.forward of the reference and its parameter gradients (sparse lattice rows included)"""
    from test_refpy_golden_gpu import check_sparse, cu, load
    from permuto_sdf import Sphere
    from permuto_sdf_b200.models import NerfHash
    G = dict(np.load(os.path.join(HERE, "golden", "refpy_golden_bg.npz")))
    m = load(NerfHash(4, Sphere(0.5, [0, 0, 0]), 1, nr_levels=24, capacity=2 ** 18), G, "bg.", 13).cuda()
    m.enable_fused()
    rgb, den = m(cu(G["bg_in.points"]), cu(G["bg_in.dirs"]), 20000)
    assert rel(rgb, G["bg_out.rgb"]) < 1e-3 and rel(den, G["bg_out.density"]) < 1e-3
    m.zero_grad()
    ((rgb * cu(G["bg_in.cb"])).sum() + (den * cu(G["bg_in.cd"])).sum()).backward()
    seen = set()
    for k, p in m.named_parameters():
        if id(p) in seen or p.grad is None:
            continue
        seen.add(id(p))
        if "lattice_values" in k:
            check_sparse(p.grad, G["bg_grad.lattice_rows"], G["bg_grad.lattice_vals"], "lattice gradient")
        else:
            assert rel(p.grad, G["bg_grad." + k]) < 1e-3, k


def _model_and_inputs(L, N, seed=0):
    from permuto_sdf import Sphere
    from permuto_sdf_b200.models import NerfHash
    torch.manual_seed(seed)
    m = NerfHash(4, Sphere(0.5, [0, 0, 0]), 1000, nr_levels=L, capacity=2 ** 16).cuda()
    with torch.no_grad():
        m.encoding.lattice_values.uniform_(-0.3, 0.3)
        for lin in [l for l in list(m.mlp_feat_and_density) + list(m.mlp_rgb) if isinstance(l, torch.nn.Linear)]:
            lin.bias.uniform_(-0.1, 0.1)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    xyz = torch.rand(N, 3, device="cuda", generator=g) * 2 - 1
    xyz = xyz / xyz.norm(dim=1, keepdim=True).clamp(min=1e-3)
    pos = torch.cat([xyz, torch.rand(N, 1, device="cuda", generator=g)], 1).contiguous()
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, device="cuda", generator=g), dim=1).contiguous()
    cb = torch.randn(N, 3, device="cuda", generator=g)
    cd = torch.randn(N, 1, device="cuda", generator=g)
    return m, pos, dirs, cb, cd


def _run(m, pos, dirs, cb, cd, it):
    m.zero_grad()
    rgb, den = m(pos, dirs, it)
    ((rgb * cb).sum() + (den * cd).sum()).backward()
    return rgb.detach().clone(), den.detach().clone(), _grads(m)


@pytest.mark.parametrize("L", [16, 24])
def test_fused_background_matches_per_op_path(cuda, L):
    """outputs within 1e-4 and every gradient within 1e-3 (relative to its largest entry) of the per-op kernels + autograd, on a sample
    count that is not a multiple of the 128-sample tile, inside the coarse-to-fine ramp"""
    m, pos, dirs, cb, cd = _model_and_inputs(L, 1000)
    ref = _run(m, pos, dirs, cb, cd, 400)
    m.enable_fused()
    out = _run(m, pos, dirs, cb, cd, 400)
    assert rel(out[0], ref[0]) < 1e-4 and rel(out[1], ref[1]) < 1e-4
    assert set(out[2]) == set(ref[2])
    for k in ref[2]:
        assert rel(out[2][k], ref[2][k]) < 1e-3, k
    with torch.no_grad():        # gradient-free evaluation (run_net_in_chunks) gives the training forward's values
        rgb, den = m(pos, dirs, 400)
    assert torch.equal(rgb, out[0]) and torch.equal(den, out[1])


def test_fused_background_deterministic(cuda):
    """deterministic mode: two backward passes give the same bits"""
    from permuto_sdf_b200._lib import call
    L = 16
    m, pos, dirs, cb, cd = _model_and_inputs(L, 3000, seed=4)
    m.enable_fused()
    call("psdf_set_deterministic", 1, L * m.encoding.capacity * 2, 64 ** 3)
    try:
        a = _run(m, pos, dirs, cb, cd, 2000)
        b = _run(m, pos, dirs, cb, cd, 2000)
    finally:
        call("psdf_set_deterministic", 0, 0, 0)
    for k in a[2]:
        assert torch.equal(a[2][k], b[2][k]), k


def _bg_trainer(direct, fused_background=True, seed=5, deterministic=False):
    """the trainer of test_direct_iteration_gpu for a scene without masks"""
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.with_mask = False
    hp.max_nr_samples_per_ray = 32
    hp.nr_samples_imp_sampling = 8
    hp.min_dist_between_samples = 1e-3
    kw = {} if fused_background is None else dict(fused_background=fused_background)
    tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=128, nr_images=4, seed=seed, optimizer="fused",
                 direct=direct, deterministic=deterministic, **kw)
    tr.set_analytic_scene()
    with torch.no_grad():       # calibration parameters start at zero: give them values so that their path is exercised
        tr.model_colorcal.weight_delta.copy_(torch.linspace(-0.2, 0.3, 12).view(4, 3))
        tr.model_colorcal.bias.copy_(torch.linspace(0.1, -0.1, 12).view(4, 3))
    return tr


def test_default_keeps_per_op_background(cuda):
    tr = _bg_trainer(None, fused_background=None)
    assert tr.execution["background"] == "per-op kernels + autograd"
    assert tr.execution["iteration"].startswith("torch.autograd")
    assert tr.model_bg.fused is None


def test_bg_compositing_matches_autograd(cuda):
    """psdf_nerf_bg_composite_* == Colorcal + sigmoid + VolumeRenderingNerf.compute_weights + integrate under autograd, on ragged packed rays
    with an empty ray and a ray of the fixed-calibration image"""
    from permuto_sdf_b200._lib import call
    from permuto_sdf_b200.models import Colorcal
    from permuto_sdf_b200.permuto_sdf import RaySamplesPacked
    counts = [5, 0, 32, 1, 17, 9]
    R, N = len(counts), sum(counts)
    se = torch.tensor([[sum(counts[:i]), sum(counts[:i + 1])] for i in range(R)], dtype=torch.int32, device="cuda")
    rsp = RaySamplesPacked(R, N)
    rsp.ray_start_end_idx = se
    g = torch.Generator(device="cuda").manual_seed(3)
    rsp.samples_dt = (torch.rand(N, 1, device="cuda", generator=g) * 0.2 + 0.01).contiguous()
    x = (torch.randn(N, 3, device="cuda", generator=g) * 2).requires_grad_(True)
    den = (torch.rand(N, 1, device="cuda", generator=g) * 5).requires_grad_(True)
    cal = Colorcal(4, 0)
    with torch.no_grad():
        cal.weight_delta.copy_(torch.randn(4, 3, device="cuda", generator=g) * 0.3)
        cal.bias.copy_(torch.randn(4, 3, device="cuda", generator=g) * 0.3)
    img = torch.tensor([1, 2, 0, 3, 2, 1], dtype=torch.int32, device="cuda")
    vr = __import__("permuto_sdf_b200.volume_rendering", fromlist=["x"]).VolumeRenderingNerf()
    rgb = torch.sigmoid(cal.calib_RGB_samples_packed(x, img, se))
    w, _, _ = vr.compute_weights(rsp, den.view(-1, 1))
    ref = vr.integrate(rsp, rgb, w)
    G = torch.randn(R, 3, device="cuda", generator=g)
    (ref * G).sum().backward()
    rsp_args = (R, N, se, 0, 0)
    head = (img, cal.weight_delta.detach(), cal.bias.detach(), 0)
    out = torch.empty(R, 3, device="cuda")
    call("psdf_nerf_bg_composite_forward", *rsp_args, x.detach(), den.detach().view(-1), rsp.samples_dt.view(-1), *head, out)
    assert rel(out, ref) < 1e-5 and float(out[1].abs().max()) == 0.0
    gx, gd = torch.zeros(N, 3, device="cuda"), torch.zeros(N, device="cuda")
    gwd, gb = torch.zeros(4, 3, device="cuda"), torch.zeros(4, 3, device="cuda")
    call("psdf_nerf_bg_composite_backward", *rsp_args, x.detach(), den.detach().view(-1), rsp.samples_dt.view(-1), *head, G, gx, gd, gwd, gb)
    assert rel(gx, x.grad) < 1e-4 and rel(gd, den.grad) < 1e-4
    assert rel(gwd, cal.weight_delta.grad) < 1e-4 and rel(gb, cal.bias.grad) < 1e-4


@pytest.mark.parametrize("it", [3000, 20000, 60000])
def test_no_mask_direct_iteration_equals_autograd_iteration(cuda, it):
    """the no-mask direct iteration (fused background, compositing, head with bg_rgb) against the autograd formulation with the same
    fused background, on identical samples and draws"""
    from test_direct_iteration_gpu import _fresh_rngs, _rays
    o, d, gt, gm, img = _rays()
    res, fixed = {}, {}

    def draw(name, fn):
        if name not in fixed:
            fixed[name] = fn()
        return fixed[name]
    for direct in (False, True):
        _fresh_rngs()
        tr = _bg_trainer(direct)
        assert tr.execution["background"] == "fused wgmma"
        assert tr.execution["iteration"].startswith("direct kernel sequence" if direct else "torch.autograd")
        tr.draw = draw
        tr.optimizer.zero_grad(set_to_none=False)
        loss = tr.forward_backward(o, d, gt, None, img, it)
        torch.cuda.synchronize()
        groups = {g["name"]: tr.optimizer.flat_grad[g["_off"]:g["_off"] + g["_n"]].clone() for g in tr.optimizer.param_groups}
        res[direct] = dict(loss=float(loss), groups=groups, lr=float(tr.last["loss_rgb"]), le=float(tr.last["loss_eikonal"]),
                           lc=float(tr.last["loss_curvature"]))
    a, b = res[True], res[False]
    assert "model_bg" in b["groups"]
    assert abs(a["loss"] - b["loss"]) <= 1e-5 * abs(b["loss"]), (a["loss"], b["loss"])
    assert abs(a["lr"] - b["lr"]) <= 1e-5 * abs(b["lr"]) and abs(a["le"] - b["le"]) <= 1e-5 * abs(b["le"]) + 1e-9
    assert abs(a["lc"] - b["lc"]) <= 1e-5 * abs(b["lc"]) + 1e-9
    for name in b["groups"]:
        assert float(b["groups"][name].abs().max()) > 0, name
        assert rel(a["groups"][name], b["groups"][name]) < 2e-4, name


def _reel():
    import scenes

    class Reel:
        pass
    rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)
    reel = Reel()
    reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
    return reel


def _train(tr, steps, graph):
    reel = _reel()
    tr.iter_nr = 20000
    if graph:
        tr.enable_cuda_graph(warmup_steps=2)
    gen = torch.Generator().manual_seed(11)
    losses = []
    for _ in range(steps):
        pix = torch.randint(0, 60 * 80, (256,), generator=gen, dtype=torch.int32).cuda()
        img = torch.randint(0, 4, (256,), generator=gen, dtype=torch.int32).cuda()
        losses.append(float(tr.step_from_reel(reel, pix, img, loss_to_host=True)))
    if graph:
        tr.disable_cuda_graph()
    return losses


def test_no_mask_direct_iteration_under_graph_replay(cuda):
    """the replayed no-mask direct iteration: finite losses, and the background table moves"""
    from test_direct_iteration_gpu import _fresh_rngs
    _fresh_rngs()
    tr = _bg_trainer(True, seed=9)
    before = tr.model_bg.encoding.lattice_values.detach().clone()
    losses = _train(tr, 8, graph=True)
    _fresh_rngs()
    assert all(np.isfinite(losses)), losses
    assert not torch.equal(before, tr.model_bg.encoding.lattice_values.detach())


def test_no_mask_deterministic_runs_are_bit_identical(cuda):
    """two deterministic no-mask runs of a few direct steps: the same losses and parameters to the bit"""
    from test_direct_iteration_gpu import _fresh_rngs
    from permuto_sdf_b200._lib import call
    out = []
    try:
        for _ in range(2):
            _fresh_rngs()
            tr = _bg_trainer(True, seed=3, deterministic=True)
            losses = _train(tr, 4, graph=False)
            out.append((losses, [p.detach().clone() for p in tr.params]))
    finally:
        call("psdf_set_deterministic", 0, 0, 0)
        _fresh_rngs()
    assert out[0][0] == out[1][0]
    for p, q in zip(out[0][1], out[1][1]):
        assert torch.equal(p, q)
