"""Volume-rendered frames on the fused kernels (Trainer.render, permuto_sdf_b200/render.py) and the render mode of the NeuS compositing
kernel (psdf_neus_render_forward, csrc/neus_fused.cu): against the reference's own VolumeRenderingNeus outputs
(tests/golden/refpy_golden.npz), bit for bit against the training instantiation of the same kernel, and against run_net_in_chunks (the
per-op mirror of the reference's renderer) on identical samples."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import scenes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rel(a, b):
    a = torch.as_tensor(a).detach().cpu().double().reshape(-1)
    b = torch.as_tensor(b).detach().cpu().double().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def render_kernel(rsp, sdf, grad, x_raw, dirs, dt, inv_s, cos_anneal, bg_rgb=None, head=(None, None, None, -1)):
    from permuto_sdf_b200._lib import call
    R = rsp[0]
    out = [torch.full((R, 3), float("nan"), device="cuda") for _ in range(3)] + [torch.full((R, 1), float("nan"), device="cuda")]
    call("psdf_neus_render_forward", *rsp, sdf, grad, x_raw, dirs, dt, inv_s, cos_anneal, *head, bg_rgb, out[0],
         out[1] if bg_rgb is not None else None, out[2], out[3])
    return out


# ------------------------------------------------------------------------------------------------ 1. kernel against the fixture
@pytest.mark.parametrize("mode", ["free", "forced"])
def test_render_kernel_matches_reference_fixture(cuda, mode):
    """VolumeRenderingNeus.compute_weights + integrate of the reference (fixture) on a ragged sample set with an empty ray: colour with the
    head on (x_raw = logit(rgb)), weights sum, background transmittance (bg_rgb = 1) and normals against fp64 normalize(sum w g)"""
    G = dict(np.load(os.path.join(HERE, "golden", "refpy_golden.npz")))
    se = cu(G["rgb_in.ray_start_end_idx"]).to(torch.int32).contiguous()
    R, N = se.shape[0], G["neus_in.sdf"].shape[0]
    rsp = (R, N, se, 0, 0)
    rgb = G["neus_in.rgb"].astype(np.float64)
    x_raw = cu(np.log(rgb / (1.0 - rgb)).astype(np.float32))
    p = "neus_%s." % mode
    inv_s = cu(G[p + "inv_s"].astype(np.float32).reshape(1))
    args = (cu(G["neus_in.sdf"]).reshape(-1), cu(G["neus_in.gradients"]), x_raw, cu(G["rgb_in.dirs"]), cu(G["neus_in.dt"]).reshape(-1), inv_s,
            float(G["neus_in.cos_anneal"]))
    pred, _, normals, wsum = render_kernel(rsp, *args)
    assert rel(pred, G[p + "pred"]) <= 1e-4 and rel(wsum, G[p + "weights_sum"]) <= 1e-4
    pred_bg_on, pred_bg, _, _ = render_kernel(rsp, *args, bg_rgb=torch.ones(R, 3, device="cuda"))
    bgT = torch.from_numpy(G[p + "bg_transmittance"]).double().reshape(-1, 1).expand(R, 3)
    assert rel(pred_bg, bgT) <= 1e-4
    assert rel(pred_bg_on, torch.from_numpy(G[p + "pred"]).double() + bgT) <= 1e-4
    # normals: fp64 F.normalize(sum_i w_i g_i) from the fixture's weights
    w = torch.from_numpy(G[p + "weights"]).double().reshape(-1, 1)
    g = torch.from_numpy(G["neus_in.gradients"]).double()
    s = se.cpu().long()
    acc = torch.zeros(R, 3, dtype=torch.float64)
    for r in range(R):
        acc[r] = (w[s[r, 0]:s[r, 1]] * g[s[r, 0]:s[r, 1]]).sum(0)
    want = F.normalize(acc, dim=1, eps=1e-12)
    assert rel(normals, want) <= 1e-4
    empty = (s[:, 1] - s[:, 0]) == 0
    assert bool(empty.any()), "the fixture has an empty ray"
    assert float(normals[empty.cuda()].abs().max()) == 0.0 and float(wsum[empty.cuda()].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ 2. render mode == training kernel
@pytest.mark.parametrize("with_bg", [False, True])
def test_render_mode_equals_training_kernel_bitwise(cuda, with_bg):
    """pred_rgb and weights_sum of the render mode are the training instantiation's, to the bit (calibrated colour head, empty rays)"""
    from permuto_sdf import OccupancyGrid, Sphere
    from permuto_sdf_b200._lib import call
    o, d = scenes.make_rays(400, seed=7)
    _, occ = scenes.analytic_occupancy(128)
    grid = OccupancyGrid(128, 1.0, [0, 0, 0])
    grid.set_grid_occupancy(cu(occ.astype(np.uint8)).bool())
    _, te, _, tx, hit = Sphere(0.5, [0, 0, 0]).ray_intersection(cu(o), cu(d))
    fg = grid.compute_samples_in_occupied_regions(cu(o), cu(d), te, tx, 1e-3, 64, True).compact_to_valid_samples()
    N, R = fg.samples_pos.shape[0], fg.ray_start_end_idx.shape[0]
    assert N > 3000 and int(((fg.ray_start_end_idx[:, 1] - fg.ray_start_end_idx[:, 0]) == 0).sum()) > 0
    g = torch.Generator(device="cuda").manual_seed(5)
    pos = fg.samples_pos
    sdf = ((pos.norm(dim=-1) - 0.3) + 0.01 * torch.randn(N, device="cuda", generator=g)).contiguous()
    grad = (F.normalize(pos, dim=-1) * (1.0 + 0.1 * torch.randn(N, 1, device="cuda", generator=g))).contiguous()
    x_raw = (torch.randn(N, 3, device="cuda", generator=g) * 2).contiguous()
    inv_s = torch.tensor([64.0], device="cuda")
    img = torch.randint(0, 4, (R,), device="cuda", generator=g, dtype=torch.int32)
    head = (img, (torch.randn(4, 3, device="cuda", generator=g) * 0.2).contiguous(), (torch.randn(4, 3, device="cuda", generator=g) * 0.2).contiguous(), 1)
    gt = torch.rand(R, 3, device="cuda", generator=g)
    mask = (torch.rand(R, device="cuda", generator=g) > 0.5).float()
    bg = torch.rand(R, 3, device="cuda", generator=g) if with_bg else None
    common = (*fg._rsp(), sdf, grad, x_raw, fg.samples_dirs, fg.samples_dt.view(-1), inv_s)
    f = lambda *s: torch.empty(*s, device="cuda")
    t_out = dict(alpha=f(N), T=f(N), pred=f(R, 3), wsum=f(R, 1), bgT=f(R, 1), loss=f(R, 3))
    tail = (t_out["alpha"], t_out["T"], None, t_out["pred"], t_out["wsum"], t_out["bgT"], t_out["loss"])
    hit_u8 = hit.reshape(-1).to(torch.uint8)
    if with_bg:
        call("psdf_neus_head_bg_loss_forward", *common, 0.35, None, gt, None, hit_u8, *head, bg, *tail)
    else:
        call("psdf_neus_head_loss_forward", *common, 0.35, None, gt, mask, hit_u8, *head, *tail)
    pred, pred_bg, normals, wsum = render_kernel(fg._rsp(), *common[5:], 0.35, bg_rgb=bg, head=head)
    assert torch.equal(pred, t_out["pred"]) and torch.equal(wsum, t_out["wsum"])
    if with_bg:
        assert torch.equal(pred_bg, t_out["bgT"] * bg)
    assert torch.isfinite(normals).all()


# ------------------------------------------------------------------------------------------------ trainers
def _trainer(L, hidden, with_mask, seed=4, deterministic=False, **kw):
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.with_mask = with_mask
    hp.max_nr_samples_per_ray = 32
    hp.nr_samples_imp_sampling = 8
    hp.min_dist_between_samples = 1e-3
    kw.setdefault("fused_background", not with_mask)
    tr = Trainer(hp, nr_levels=L, capacity=2 ** 14, sdf_hidden=hidden, occupancy_resolution=128, nr_images=4, seed=seed, optimizer="fused",
                 deterministic=deterministic, **kw)
    tr.set_analytic_scene()
    return tr


def _reel_rays(n):
    from test_direct_iteration_gpu import _rays
    return _rays(n)


def _trained(L, hidden, with_mask, steps=3):
    """a fitted scene: the sphere-fit phase, a few training steps at iteration 20000 (every lattice level active; the first step refreshes
    part of the occupancy grid from the model), then one more occupancy refresh; models in eval() (no jitter)"""
    from test_direct_iteration_gpu import _fresh_rngs
    _fresh_rngs()
    tr = _trainer(L, hidden, with_mask)
    tr.fit_sphere(200)
    tr.iter_nr = 20000
    o, d, gt, gm, img = _reel_rays(256)
    for _ in range(steps):
        tr.step(o, d, gt, gm, img)
    tr.update_occupancy(tr.iter_nr)
    for m in (tr.model_sdf, tr.model_rgb, tr.model_bg):
        if m is not None:
            m.eval()
    return tr


def _schedule(tr):
    """cos_anneal_ratio and forced variance of the trainer's iteration (Trainer.losses)"""
    from permuto_sdf_b200.models import map_range_val
    it, hp = tr.iter_nr, tr.hp
    return map_range_val(it, 0.0, hp.forced_variance_finish_iter, 0.0, 1.0), map_range_val(it, 0.0, hp.forced_variance_finish_iter, 0.3,
                                                                                            hp.forced_variance_finish)


def _frame_rays(R, seed):
    """camera rays (10% miss the bounding sphere) plus rays that cross the bounding sphere outside the occupied shell"""
    o, d = scenes.make_rays(R, seed=seed)
    n_empty = R // 20
    o[:n_empty] = np.stack([np.full(n_empty, 0.44, np.float32), np.linspace(-0.1, 0.1, n_empty, dtype=np.float32),
                            np.full(n_empty, 1.2, np.float32)], 1)
    d[:n_empty] = np.array([0.0, 0.0, -1.0], np.float32)
    return cu(o), cu(d)


@pytest.mark.parametrize("L,hidden", [(16, 32), (16, 64), (24, 32), (24, 64)])
@pytest.mark.parametrize("with_mask", [True, False])
def test_render_matches_run_net_in_chunks(cuda, L, hidden, with_mask):
    """same samples; the differences come from the fused SDF value, gradient and geometric feature and the order of the compositing sums.
    A ray that points away from a bounding sphere it intersects behind its origin gets non-finite background samples in both paths
    (RaySampler.compute_samples_bg): the two must agree on which rays those are."""
    from permuto_sdf_b200.train import run_net_in_chunks
    tr = _trained(L, hidden, with_mask)
    o, d = _frame_rays(3000, seed=11)
    it = tr.iter_nr
    cos, fv = _schedule(tr)
    ref = run_net_in_chunks(o, d, 1000, with_mask, tr.hp, tr.model_sdf, tr.model_rgb, tr.model_bg, tr.occupancy_grid, it, cos, fv)
    out = tr.render(o, d, 1000, it, cos, fv)
    assert (out[1] is None) == (ref[1] is None) == with_mask
    wsum = ref[3].view(-1)
    assert int((wsum > 0.5).sum()) > 100 and int((wsum == 0).sum()) > 100, "frame must have opaque rays and rays without samples"
    fin = torch.isfinite(ref[0]).all(1)
    assert torch.equal(fin, torch.isfinite(out[0]).all(1))
    err = {k: float((a[fin] - b[fin]).abs().max()) for k, a, b in zip(("rgb", "bg", "normals", "wsum"), out, ref) if b is not None}
    assert err["rgb"] <= 1e-4 and err["wsum"] <= 1e-4 and err.get("bg", 0.0) <= 1e-4, err
    sel = wsum > 1e-3
    assert float((out[2][sel] - ref[2][sel]).abs().max()) <= 1e-3, err
    assert float(out[2][wsum == 0].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ 4. chunk-size invariance
@pytest.mark.parametrize("with_mask", [True, False])
def test_render_chunk_size_invariance(cuda, with_mask):
    """chunks of 997 and 4096 rays and the whole frame in one chunk give the same bits; the first chunks of the 997 split have no sample at all"""
    tr = _trained(16, 64, with_mask)
    o, d = _frame_rays(6000, seed=12)
    miss = 2000
    o[:miss] = torch.tensor([0.0, 0.0, 1.2], device="cuda")
    d[:miss] = torch.tensor([0.0, 1.0, 0.0], device="cuda")       # parallel to the bounding sphere, outside it
    outs = [tr.render(o, d, c, tr.iter_nr, *_schedule(tr)) for c in (997, 4096, 6000)]
    assert float(outs[0][3][:miss].abs().max()) == 0.0
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert (a is None) == (b is None)
            if a is not None:
                assert torch.equal(a.view(torch.int32), b.view(torch.int32))      # bit patterns (non-finite background rays included)


# ------------------------------------------------------------------------------------------------ 5. no side effects
def _state(tr):
    from permuto_sdf import OccupancyGrid, RaySampler, VolumeRendering
    g = tr.occupancy_grid
    return dict(params=[p.detach().clone() for p in tr.params], grads=[None if p.grad is None else p.grad.clone() for p in tr.params],
                grid=(g.get_grid_values().clone(), g.get_grid_occupancy().clone()),
                rng=[(r.state, r.inc) for r in (OccupancyGrid.m_rng, RaySampler.m_rng, VolumeRendering.m_rng)],
                torch_rng=(torch.get_rng_state(), torch.cuda.get_rng_state()), counters=(tr.iter_nr, tr.sphere_fit_iter))


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return a == b


@pytest.mark.parametrize("with_mask", [True, False])
def test_render_has_no_side_effects(cuda, with_mask):
    """deterministic mode: step, render (models in eval() around it), step gives the losses and parameters of step, step; render leaves
    parameters, .grad, the occupancy grid, the generators and the counters untouched"""
    from test_direct_iteration_gpu import _fresh_rngs
    from permuto_sdf_b200._lib import call
    o, d, gt, gm, img = _reel_rays(256)
    fo, fd = _frame_rays(2000, seed=13)
    runs = []
    try:
        for with_render in (False, True):
            _fresh_rngs()
            torch.manual_seed(0)
            tr = _trainer(16, 64, with_mask, deterministic=True)
            losses = [float(tr.step(o, d, gt, gm, img))]
            if with_render:
                models = [m for m in (tr.model_sdf, tr.model_rgb, tr.model_bg) if m is not None]
                for m in models:
                    m.eval()
                before = _state(tr)
                tr.render(fo, fd, 700, tr.iter_nr, 1.0, 0.8)
                torch.cuda.synchronize()
                assert _same(before, _state(tr))
                for m in models:
                    m.train()
            losses.append(float(tr.step(o, d, gt, gm, img)))
            runs.append((losses, [p.detach().clone() for p in tr.params]))
    finally:
        call("psdf_set_deterministic", 0, 0, 0)
        _fresh_rngs()
    assert runs[0][0] == runs[1][0]
    assert all(torch.equal(p, q) for p, q in zip(runs[0][1], runs[1][1]))


# ------------------------------------------------------------------------------------------------ 6. refusals
def test_render_refuses_configurations_off_the_fused_kernels(cuda):
    o, d = _frame_rays(64, seed=1)
    tr = _trainer(16, 64, True, fused_inference=False)
    with pytest.raises(RuntimeError, match="SDF model is not on the fused kernels"):
        tr.render(o, d)
    tr = _trainer(16, 64, False, fused_background=False)
    with pytest.raises(RuntimeError, match="background model"):
        tr.render(o, d)
    from permuto_sdf_b200.render import VolumeRender
    tr = _trainer(16, 64, True)
    with pytest.raises(ValueError, match="chunk_size"):
        tr.render(o, d, chunk_size=VolumeRender.max_chunk(tr.hp) + 1)
