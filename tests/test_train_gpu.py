"""GPU tests of the hot-path drivers: SDF + gradient parity against the CPU oracle (<= 1e-3 relative, the
north-star tolerance), NeuS weights against the oracle formula, one full training iteration, importance
resampling driver, sphere tracing on an analytic scene."""
import numpy as np
import pytest
import torch

import scenes
from oracle import encoding_oracle as eo

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.fixture(scope="module")
def trainer(cuda):
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.max_nr_samples_per_ray = 32
    hp.nr_samples_imp_sampling = 8
    hp.min_dist_between_samples = 1e-3
    tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=128, nr_images=4, seed=1)
    tr.set_analytic_scene()
    return tr


def test_sdf_and_gradient_match_oracle(trainer):
    m = trainer.model_sdf
    torch.manual_seed(0)
    pos = (torch.rand(3000, 3) - 0.5) * 0.8
    it = 2000
    sdf, grad, geom = m.get_sdf_and_gradient(pos.cuda(), it)
    enc = m.encoding
    lin = [l for l in m.mlp_sdf if isinstance(l, torch.nn.Linear)]
    W = [l.weight.detach().cpu() for l in lin]; B = [l.bias.detach().cpu() for l in lin]
    window = eo.coarse2fine(enc.nr_levels, 0.3 + 0.7 * it / m.nr_iters_for_c2f)
    s0, g0, f0 = eo.sdf_and_gradient(pos, enc.lattice_values.detach().cpu(), enc.scale_factor.cpu(), enc.random_shift_per_level.detach().cpu(),
                                     window, W, B, True, 1e-3)
    assert rel(sdf, s0) < 1e-3 and rel(grad, g0) < 1e-3 and rel(geom, f0) < 1e-3
    # finite-difference variant of the reference API
    s1, g1, _ = m.get_sdf_and_gradient(pos.cuda(), it, method="finite_difference")
    assert rel(s1, s0) < 1e-3
    # gradient-free evaluations are routed through the fused tensor-core kernel
    assert getattr(m, "fused", None) is not None
    with torch.no_grad():
        s2, f2 = m(pos.cuda(), it)
    assert rel(s2, s0) < 1e-3 and rel(f2, f0) < 1e-3


def test_neus_weights_match_oracle(trainer):
    from permuto_sdf import OccupancyGrid
    o, d = scenes.make_rays(128, seed=2)
    to, td = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    _, te, _, tx, _ = trainer.aabb.ray_intersection(to, td)
    rsp = trainer.occupancy_grid.compute_samples_in_occupied_regions(to, td, te, tx, 1e-3, 48, False).compact_to_valid_samples()
    n = rsp.samples_pos.shape[0]
    sdf = (rsp.samples_pos.norm(dim=1, keepdim=True) - 0.3).requires_grad_(True)
    grads = torch.nn.functional.normalize(rsp.samples_pos, dim=1).requires_grad_(True)
    vr = trainer.model_rgb.volume_renderer_neus
    w, wsum, bg, inv_s = vr.compute_weights(rsp, sdf, grads, 0.5, forced_variance=0.5)
    a0 = eo.neus_alpha(sdf.detach().cpu(), grads.detach().cpu(), rsp.samples_dirs.cpu(), rsp.samples_dt.cpu(), float(np.exp(5.0)), 0.5)
    se = rsp.ray_start_end_idx.cpu().numpy()
    w0 = torch.zeros(n, 1)
    for s, e in se:
        if e > s:
            T = torch.cumprod(torch.cat([torch.ones(1, 1), (1 - a0[s:e - 1] + 1e-7)], 0), 0)
            w0[s:e] = a0[s:e] * T
    assert rel(w, w0) < 1e-3
    assert torch.allclose(wsum.cpu()[:, 0], torch.tensor([float(w0[s:e].sum()) for s, e in se]), atol=1e-4)
    # gradient flows through the hand-written backward kernels
    col = torch.rand(n, 3, device="cuda", requires_grad=True)
    pred = vr.integrate(rsp, col, w)
    (pred.sum() + wsum.sum() + bg.sum()).backward()
    assert sdf.grad.abs().sum() > 0 and col.grad.abs().sum() > 0 and grads.grad.abs().sum() > 0


def test_full_training_iterations(trainer):
    from permuto_sdf import PermutoSDF

    class Reel:
        pass
    rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)
    reel = Reel()
    reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
    before = trainer.model_sdf.encoding.lattice_values.detach().clone()
    losses = []
    for i in range(3):
        o, d, gt, gm, img = PermutoSDF.random_rays_from_reel(reel, 256)
        losses.append(float(trainer.step(o, d, gt, gm, img)))
    assert all(np.isfinite(l) for l in losses)
    assert trainer.last["nr_samples"] > 1000
    assert not torch.equal(before, trainer.model_sdf.encoding.lattice_values.detach()), "optimizer did not update the SDF lattice"
    for name, p in trainer.model_sdf.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), name
    assert trainer.model_rgb.encoding.lattice_values.grad.abs().sum() > 0
    occ = trainer.occupancy_grid.get_grid_occupancy()
    assert occ.dtype == torch.bool and 0 < int(occ.sum()) < occ.numel()


def test_sphere_trace_analytic(cuda):
    """sphere tracing an exact sphere SDF (a stand-in model with the reference's model interface)"""
    from permuto_sdf import OccupancyGrid, Sphere
    from permuto_sdf_b200.train import sphere_trace

    class AnalyticSDF(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.boundary_primitive = Sphere(0.5, [0, 0, 0])
            self.last_iter_nr = 0

        def forward(self, p, it):
            return p.norm(dim=1, keepdim=True) - 0.3, None

        def get_sdf_and_gradient(self, p, it):
            p.requires_grad_(True)
            s = p.norm(dim=1, keepdim=True) - 0.3
            return s, torch.autograd.grad(s.sum(), p)[0], None
    grid = OccupancyGrid(128, 1.0, [0, 0, 0])
    pts = grid.compute_grid_points(False)
    grid.update_with_sdf((pts.norm(dim=1, keepdim=True) - 0.3).contiguous(), 512.0, 1e10, 1e-4)
    o, d = scenes.make_rays(2000, seed=9, miss_fraction=0.2, axis_aligned=0)
    to, td = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    model = AnalyticSDF()
    pts, sdf, grads, _, rsp = sphere_trace(30, to, td, model, True, 0.9, 2e-4, grid)
    n = rsp.ray_start_end_idx[:, 1] - rsp.ray_start_end_idx[:, 0]
    assert int(n.sum()) == pts.shape[0] and pts.shape[0] > 500
    r = pts.norm(dim=1)
    assert float((r - 0.3).abs().median()) < 5e-4, "traced points should sit on the analytic surface"
    # exact ray / sphere hit for comparison
    oo, dd = to[n > 0], td[n > 0]
    b = (oo * dd).sum(1); c = (oo * oo).sum(1) - 0.09
    disc = b * b - c
    ok = disc > 1e-4
    t = -b - torch.sqrt(disc.clamp(min=0))
    hitp = oo + t[:, None] * dd
    assert float((pts[ok] - hitp[ok]).norm(dim=1).median()) < 2e-3
    # without a grid: one sample per ray
    pts2, _, _, _, rsp2 = sphere_trace(30, to, td, model, False, 0.9, 2e-4, None)
    assert pts2.shape[0] == 2000 and rsp2.rays_have_equal_nr_of_samples


@pytest.mark.parametrize("it,tol_grad", [(60000, 1e-3), (3000, 6e-2)])
def test_fused_render_loss_equals_modular_iteration(trainer, it, tol_grad):
    """one whole iteration (sampling -> models -> compositing -> losses -> backward) with the fused NeuS compositing + loss (+ curvature)
    kernels against the same iteration on the per-op kernels + torch losses; identical samples (RNG states restored).
    Iteration 60000 is past the curvature phase: everything agrees to 1e-3. At iteration 3000 the curvature term is active; it is
    acos(n . n') / pi for normals 1e-4 apart, i.e. acos within 1e-6 of 1 where its condition number is ~1e6: fp32 rounding of the dot
    product (FMA or not) moves the term and its gradient by percents in ANY implementation, so the gradients are compared at 6e-2."""
    from permuto_sdf import OccupancyGrid, PermutoSDF, RaySampler, VolumeRendering

    class Reel:
        pass
    rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)
    reel = Reel()
    reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
    o, d, gt, gm, img = PermutoSDF.random_rays_from_reel(reel, 256)
    rngs = [OccupancyGrid.m_rng, RaySampler.m_rng, VolumeRendering.m_rng]
    states = [(r.state, r.inc) for r in rngs]
    tstate, cstate = torch.get_rng_state(), torch.cuda.get_rng_state()
    res = {}
    for mode in (True, False):
        for r, (s, i) in zip(rngs, states):
            r.state, r.inc = s, i
        torch.set_rng_state(tstate); torch.cuda.set_rng_state(cstate)
        trainer.fused_render = mode
        trainer.optimizer.zero_grad(set_to_none=False)
        loss = trainer.losses(o, d, gt, gm, img, it)
        loss.backward()
        res[mode] = (float(loss), trainer.last["nr_samples"], trainer.model_sdf.encoding.lattice_values.grad.clone(),
                     trainer.model_rgb.encoding.lattice_values.grad.clone(), trainer.model_rgb.mlp.layers[0].weight.grad.clone()
                     if hasattr(trainer.model_rgb.mlp, "layers") else None)
    trainer.fused_render = True
    assert res[True][1] == res[False][1] and res[True][1] > 1000
    assert abs(res[True][0] - res[False][0]) / abs(res[False][0]) < (1e-4 if tol_grad <= 1e-3 else 1e-3)
    assert rel(res[True][2], res[False][2]) < tol_grad
    assert rel(res[True][3], res[False][3]) < 1e-3


@pytest.mark.parametrize("with_grid", [True, False])
def test_fused_sphere_trace_equals_masked_loop(trainer, with_grid):
    """the single-kernel sphere tracer against the reference-style masked gather / scatter loop on the same network: identical
    traced points (bit for bit), on a freshly initialised SDF (sphere of radius ~0.3 from geometric init is not needed: any field works)"""
    import permuto_sdf_b200.train as tr
    o, d = scenes.make_rays(3000, seed=21, miss_fraction=0.2, axis_aligned=0)
    to, td = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    m = trainer.model_sdf
    m.last_iter_nr = 20000
    with torch.no_grad():       # an SDF-like field: bias the output so that rays do converge somewhere inside the sphere
        lin = [l for l in m.mlp_sdf if isinstance(l, torch.nn.Linear)]
        lin[-1].bias[0] = 0.05
    grid = trainer.occupancy_grid if with_grid else None
    res = {}
    for fused in (False, True):
        tr.FUSED_SPHERE_TRACE = fused
        with torch.no_grad():           # rendering context: the loop's network evaluations take the same fused tensor-core path
            pts, sdf, grads, geom, rsp = tr.sphere_trace(12, to, td, m, True, 0.9, 1e-3, grid)
        res[fused] = (pts.clone(), sdf.clone(), grads.clone())
    tr.FUSED_SPHERE_TRACE = True
    assert res[True][0].shape == res[False][0].shape and res[True][0].shape[0] > 500
    assert torch.equal(res[True][0], res[False][0]), float((res[True][0] - res[False][0]).abs().max())
    assert torch.equal(res[True][1], res[False][1])
    assert torch.equal(rsp.samples_pos, res[True][0])


def test_reference_default_sizes_iteration(cuda):
    """the reference's own network sizes (24 levels, 32-wide SDF MLP: models.py:131-160, 309-340) go through the fused kernels too"""
    from permuto_sdf import PermutoSDF
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.max_nr_samples_per_ray = 32
    hp.nr_samples_imp_sampling = 8
    hp.min_dist_between_samples = 1e-3
    tr = Trainer(hp, nr_levels=24, capacity=2 ** 15, sdf_hidden=32, occupancy_resolution=64, nr_images=4, seed=2, optimizer="fused")
    tr.set_analytic_scene()
    assert tr.model_sdf.fused is not None and tr.model_sdf.fused_training and tr.model_rgb.fused is not None

    class Reel:
        pass
    rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)
    reel = Reel()
    reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
    before = [p.detach().clone() for p in tr.params]
    for i in range(2):
        o, d, gt, gm, img = PermutoSDF.random_rays_from_reel(reel, 256)
        loss = float(tr.step(o, d, gt, gm, img))
        assert np.isfinite(loss)
    moved = [float((a - b.detach()).abs().max()) for a, b in zip(before, tr.params)]
    assert max(moved) > 0 and all(np.isfinite(m) for m in moved)


@pytest.mark.parametrize("graph", [False, True])
def test_iteration_with_background_model(cuda, graph):
    """--no mask path (train_permuto_sdf.py:155-171): NeRF++ background model composited behind the SDF foreground; the fused NeuS
    kernel blends bg_transmittance * bg_rgb and hands its gradient back to the background network; also under CUDA-graph replay"""
    from permuto_sdf import PermutoSDF
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.with_mask = False
    hp.max_nr_samples_per_ray = 24
    hp.nr_samples_imp_sampling = 8
    hp.nr_samples_bg = 16
    hp.min_dist_between_samples = 1e-3
    tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=32, occupancy_resolution=64, nr_images=4, seed=5, optimizer="fused")
    tr.set_analytic_scene()
    assert tr.model_bg is not None
    if graph:
        tr.enable_cuda_graph(warmup_steps=1)

    class Reel:
        pass
    rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)
    reel = Reel()
    reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
    bg0 = tr.model_bg.encoding.lattice_values.detach().clone()
    gen = torch.Generator().manual_seed(3)
    losses = []
    for i in range(4):
        pix = torch.randint(0, 60 * 80, (256,), generator=gen, dtype=torch.int32).cuda()
        img = torch.randint(0, 4, (256,), generator=gen, dtype=torch.int32).cuda()
        with torch.no_grad():
            o, d, gt, gm, idx = PermutoSDF.rays_from_reel_indices(reel, pix, img)
        losses.append(float(tr.step(o, d, gt, gm, idx)))
    tr.disable_cuda_graph()
    from permuto_sdf import OccupancyGrid, RaySampler, RaySamplesPacked, VolumeRendering
    RaySamplesPacked.static_capacity = False
    assert all(np.isfinite(l) for l in losses), losses
    assert not torch.equal(bg0, tr.model_bg.encoding.lattice_values.detach()), "the background model received no gradient"


def test_flat_optimizer_with_modular_sdf_path_matches_adamw_gradients(cuda):
    """ADVICE r1: optimizer='fused' turns on grad_in_place; on the modular SDF path (fused_training=False) the create_graph backward
    of get_sdf_and_gradient must NOT scatter d(sum sdf)/d(lattice) into lattice.grad. Gradients of one iteration must equal the
    ones of the plain torch.optim.AdamW configuration."""
    from permuto_sdf import PermutoSDF, RaySamplesPacked
    from permuto_sdf_b200.train import HyperParams, Trainer
    import test_graph_gpu
    grads = {}
    for opt in ("adamw", "fused"):
        test_graph_gpu._fresh_rngs()
        hp = HyperParams()
        hp.max_nr_samples_per_ray = 32
        hp.nr_samples_imp_sampling = 8
        hp.min_dist_between_samples = 1e-3
        hp.offsurface_weight = 0.0
        tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=128, nr_images=4, seed=4, optimizer=opt,
                     fused_training=False, fused_render=False)
        assert tr.execution["sdf_training"].startswith("per-op")
        tr.set_analytic_scene()
        tr.iter_nr = 60000            # past the curvature phase (its random directions come from torch's generator)
        rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)

        class Reel:
            pass
        reel = Reel()
        reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
        gen = torch.Generator().manual_seed(5)
        pix = torch.randint(0, 60 * 80, (256,), generator=gen, dtype=torch.int32).cuda()
        img = torch.randint(0, 4, (256,), generator=gen, dtype=torch.int32).cuda()
        with torch.no_grad():
            o, d, gt, gm, idx = PermutoSDF.rays_from_reel_indices(reel, pix, img)
        tr.step(o, d, gt, gm, idx, update_occupancy=False, optimizer_step=False)
        grads[opt] = torch.cat([p.grad.detach().reshape(-1).clone() for p in tr.model_sdf.parameters() if p.grad is not None])
    test_graph_gpu._fresh_rngs()
    a, b = grads["adamw"], grads["fused"]
    assert a.shape == b.shape and float(a.norm()) > 0
    assert float((a - b).norm() / a.norm()) < 1e-3


def test_trainer_checkpoint_roundtrip_and_chunked_render(cuda, tmp_path):
    """f4: Trainer.save writes the reference's file layout (train_permuto_sdf.py:444-453), Trainer.load restores a run exactly
    (next loss identical), run_net_in_chunks (train_permuto_sdf.py:172-209) equals the one-shot render"""
    import os
    from permuto_sdf_b200.train import HyperParams, Trainer, run_net, run_net_in_chunks
    import test_graph_gpu

    def make():
        test_graph_gpu._fresh_rngs()
        hp = HyperParams()
        hp.max_nr_samples_per_ray = 32
        hp.nr_samples_imp_sampling = 8
        hp.min_dist_between_samples = 1e-3
        tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=64, nr_images=4, seed=6, optimizer="fused")
        tr.set_analytic_scene()
        tr.iter_nr = 60000
        return tr
    o, d = scenes.make_rays(256, seed=3)
    o, d = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    gt, gm = torch.rand(256, 3, device="cuda"), torch.ones(256, 1, device="cuda")
    img = torch.zeros(256, dtype=torch.int32, device="cuda")
    tr = make()
    for _ in range(3):
        tr.step(o, d, gt, gm, img, update_occupancy=True)
    path = tr.save(str(tmp_path), "run")
    assert sorted(os.listdir(path)) == ["colorcal_model.pt", "grid_occupancy.pt", "grid_values.pt", "rgb_model.pt", "sdf_model.pt", "trainer_state.pt"]
    assert path.endswith(os.path.join("run", "60003", "models"))
    tr2 = make()
    tr2.load(path)
    assert tr2.iter_nr == tr.iter_nr and tr2.optimizer.step_count == tr.optimizer.step_count
    for a, b in zip(tr.params, tr2.params):
        assert torch.equal(a, b)
    assert torch.equal(tr.occupancy_grid.get_grid_occupancy(), tr2.occupancy_grid.get_grid_occupancy())
    # same state -> same evaluation (eval mode: no jitter)
    for t in (tr, tr2):
        t.model_sdf.eval(); t.model_rgb.eval()
    with torch.no_grad():
        full = [run_net(True, t.hp, o, d, None, t.model_sdf, t.model_rgb, None, None, t.occupancy_grid, 60003, 1.0, 0.8) for t in (tr, tr2)]
    assert torch.equal(full[0][0], full[1][0])
    rgb_c, bg_c, nrm_c, ws_c = run_net_in_chunks(o, d, 100, True, tr.hp, tr.model_sdf, tr.model_rgb, None, tr.occupancy_grid, 60003, 1.0, 0.8)
    assert bg_c is None and rgb_c.shape == (256, 3)
    assert float((rgb_c - full[0][0]).abs().max()) < 1e-5 and float((ws_c - full[0][4]).abs().max()) < 1e-5
    test_graph_gpu._fresh_rngs()


def test_deterministic_mode_reproduces_training_bits(cuda):
    """Trainer(deterministic=True): two runs of the direct iteration from the same seed and inputs (occupancy refresh included) give
    bit-identical losses, gradients and parameters -- the fixed-point gradient reductions do not depend on the order of the atomics"""
    from permuto_sdf import OccupancyGrid, RaySampler, VolumeRendering
    from permuto_sdf_b200.train import HyperParams, Trainer
    g = torch.Generator().manual_seed(7)
    pix = [torch.randint(0, 32 * 32, (256,), generator=g, dtype=torch.int32).cuda() for _ in range(3)]
    img = [torch.randint(0, 2, (256,), generator=g, dtype=torch.int32).cuda() for _ in range(3)]
    rgb, mask, K, tf = (torch.from_numpy(a).cuda() for a in scenes.synthetic_reel(nimg=2, H=32, W=32))

    class Reel:
        rgb_reel, mask_reel, K_reel, tf_world_cam_reel = rgb, mask, K, tf

    def run():
        for c in (OccupancyGrid, RaySampler, VolumeRendering):      # the class generators start from their initial state
            c.m_rng.to_host()
            fresh = type(c.m_rng)()
            c.m_rng.state, c.m_rng.inc = fresh.state, fresh.inc
        hp = HyperParams()
        hp.nr_rays = 256
        tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=32, nr_images=2, occupancy_resolution=64, seed=3, optimizer="fused",
                     deterministic=True)
        tr.set_analytic_scene()
        tr.iter_nr = 20000
        out = []
        for i in range(3):
            loss = tr.step_from_reel(Reel, pix[i], img[i], update_occupancy=True, optimizer_step=False)
            torch.cuda.synchronize()
            out.append(torch.tensor([float(loss)]))
            out += [p.grad.detach().clone() for p in tr.params if p.grad is not None]
            tr.optimizer_step()
        out += [p.detach().clone() for p in tr.params] + [tr.occupancy_grid.get_grid_values().clone()]
        return out

    try:
        a, b = run(), run()
    finally:
        from permuto_sdf_b200._lib import call
        call("psdf_set_deterministic", 0, 0, 0)
    assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))
