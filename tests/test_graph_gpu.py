"""CUDA-graph replay of the training iteration (Trainer.enable_cuda_graph): static-capacity containers, device-resident pcg32
generators / iteration number / AdamW step must give the same trajectory as eager iterations with exactly-sized containers.
Curvature and off-surface terms draw from torch's Philox generator, whose offsets differ under capture, so the comparison
runs past the curvature phase with the off-surface weight at zero; everything else (samplers, jitter, importance resampling,
compositing, losses, optimizer, occupancy refresh) is driven by the pcg32 streams and is reproducible."""
import numpy as np
import pytest
import torch

import scenes

pytestmark = pytest.mark.gpu


def _fresh_rngs():
    from permuto_sdf import OccupancyGrid, RaySampler, RaySamplesPacked, VolumeRendering
    from permuto_sdf_b200.permuto_sdf import _Pcg32Host
    OccupancyGrid.m_rng, RaySampler.m_rng, VolumeRendering.m_rng = _Pcg32Host(), _Pcg32Host(), _Pcg32Host()
    RaySamplesPacked.static_capacity = False


def _run(mode, steps=8, start_iter=60000, lr=None, grad_at_last=False):
    from permuto_sdf import PermutoSDF
    from permuto_sdf_b200.train import HyperParams, Trainer
    _fresh_rngs()
    hp = HyperParams()
    hp.max_nr_samples_per_ray = 32
    hp.nr_samples_imp_sampling = 8
    hp.min_dist_between_samples = 1e-3
    hp.offsurface_weight = 0.0
    if lr is not None:
        hp.lr = lr
    tr = Trainer(hp, nr_levels=8, capacity=2 ** 14, sdf_hidden=64, occupancy_resolution=128, nr_images=4, seed=3, optimizer="fused")
    tr.set_analytic_scene()
    tr.iter_nr = start_iter
    if mode == "graph":
        tr.enable_cuda_graph(warmup_steps=2)

    class Reel:
        pass
    rgb, mask, K, tf = scenes.synthetic_reel(nimg=4, H=60, W=80)
    reel = Reel()
    reel.rgb_reel, reel.mask_reel, reel.K_reel, reel.tf_world_cam_reel = [torch.from_numpy(a).cuda() for a in (rgb, mask, K, tf)]
    gen = torch.Generator().manual_seed(11)
    losses, counts = [], []
    for i in range(steps):
        pix = torch.randint(0, 60 * 80, (256,), generator=gen, dtype=torch.int32).cuda()
        img = torch.randint(0, 4, (256,), generator=gen, dtype=torch.int32).cuda()
        last = grad_at_last and i == steps - 1
        if mode == "graph":         # indices in, ray generation captured with the iteration
            losses.append(float(tr.step_from_reel(reel, pix, img, optimizer_step=not last)))
        else:
            with torch.no_grad():
                o, d, gt, gm, idx = PermutoSDF.rays_from_reel_indices(reel, pix, img)
            losses.append(float(tr.step(o, d, gt, gm, idx, optimizer_step=not last)))
        counts.append(int(tr.last["nr_samples_dev"]))
    params = [p.detach().clone() for p in tr.params]
    grad = tr.optimizer.flat_grad.detach().clone()
    launches = tr.graph_launches_per_step()
    tr.disable_cuda_graph()
    _fresh_rngs()
    return losses, counts, params, launches, grad


def test_graph_replay_reproduces_eager_iterations(cuda):
    """learning rate 0 keeps the parameters fixed, so every iteration (sampling, jitter, importance resampling, models,
    compositing, losses, backward) must agree between eager exact-size containers and replayed graphs with static capacity"""
    l_e, n_e, _, _, g_e = _run("eager", lr=0.0, grad_at_last=True)
    l_g, n_g, _, launches, g_g = _run("graph", lr=0.0, grad_at_last=True)
    assert n_e == n_g, "static-capacity containers must hold the same samples: %s vs %s" % (n_e, n_g)
    assert launches is not None and launches > 10
    for a, b in zip(l_e, l_g):
        assert abs(a - b) / abs(a) < 1e-4, (l_e, l_g)
    # gradient of a replayed iteration (the 6th after capture) against the eager one: same up to accumulation order
    assert float(g_e.abs().max()) > 0
    assert float((g_e - g_g).norm() / g_e.norm()) < 1e-3


def test_graph_training_trajectory(cuda):
    """with the real learning rate both modes train: losses finite and decreasing over the 8 iterations, similar sample counts,
    parameters moved by the replayed optimizer graph. The two loss sequences are NOT compared value by value: any last-bit difference
    between the two formulations becomes a full +-lr step of Adam (eps = 1e-15) for a near-zero gradient, and the sequences drift from
    there. Exact equivalence of the replayed iteration -- samples, losses,
    gradients -- is what test_graph_replay_reproduces_eager_iterations (lr = 0) and test_fused_adamw_device_step_under_cuda_graph check."""
    l_e, n_e, p_e, _, _ = _run("eager")
    l_g, n_g, p_g, _, _ = _run("graph")
    for l in (l_e, l_g):
        assert all(np.isfinite(l)) and l[-1] < l[0], l
    assert abs(l_e[0] - l_g[0]) / abs(l_e[0]) < 1e-4, "the first iteration starts from identical parameters"
    assert max(abs(a - b) for a, b in zip(n_e, n_g)) <= 0.05 * max(n_e)
    p_0 = _run("eager", steps=0)[2]
    moved = sum(float(((a - b) ** 2).sum()) for a, b in zip(p_g, p_0)) ** 0.5
    assert moved > 1e-2, "the replayed optimizer graph must move the parameters"


def test_graph_recaptures_when_schedule_branch_changes(cuda):
    """crossing a schedule boundary (end of the curvature phase at iteration 51001) invalidates the captured graph"""
    l, n, _, _, _ = _run("graph", steps=7, start_iter=50997)
    assert all(np.isfinite(l)) and min(n) > 1000
