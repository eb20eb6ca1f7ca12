"""One small invocation of the hot path on cuda:0, checked against the oracle (the only product-side file
that is allowed to import oracle/, as the checker -- see __graft_entry__.smoke)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(verbose=True):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    if not torch.cuda.is_available():
        raise RuntimeError("smoke() needs a CUDA device; there is no CPU path")
    from oracle import encoding_oracle as eo
    from oracle import rayops as orc
    from permuto_sdf_b200 import load_library
    from permuto_sdf_b200 import permutohedral_encoding as pe
    from permuto_sdf_b200.permuto_sdf import OccupancyGrid, Sphere
    from permuto_sdf_b200.train import HyperParams, Trainer

    lib = load_library()
    assert lib.psdf_device_ok() == 1, "libpsdf_b200.so is loaded but no sm_90 (H100) device is visible"
    torch.cuda.set_device(0)
    torch.manual_seed(0)

    # 1. encoding forward + positions gradient against the CPU oracle
    enc = pe.PermutoEncoding(3, 2 ** 14, 4, 2, np.geomspace(1.0, 1e-2, 4), concat_points=True, concat_points_scaling=1e-3, init_scale=1.0)
    pos = (torch.rand(2048, 3) - 0.5)
    p = pos.cuda().requires_grad_(True)
    out = enc(p)
    (g,) = torch.autograd.grad(out.sum(), p)
    pc = pos.clone().requires_grad_(True)
    ref = eo.encode(pc, enc.lattice_values.detach().cpu(), enc.scale_factor.cpu(), enc.random_shift_per_level.detach().cpu(), None, True, 1e-3)
    (gr,) = torch.autograd.grad(ref.sum(), pc)
    e1 = float((out.detach().cpu() - ref.detach()).abs().max() / ref.detach().abs().max())
    e2 = float((g.cpu() - gr).abs().max() / gr.abs().max())
    assert e1 < 1e-4 and e2 < 1e-3, ("encoding parity", e1, e2)

    # 2. occupancy-grid ray sampling against the C oracle (bit exact indices)
    V = 64
    rng = np.random.RandomState(0)
    cam = rng.randn(256, 3); cam = 1.2 * cam / np.linalg.norm(cam, axis=1, keepdims=True)
    tgt = rng.uniform(-0.3, 0.3, (256, 3))
    d = tgt - cam; d /= np.linalg.norm(d, axis=1, keepdims=True)
    o, d = cam.astype(np.float32), d.astype(np.float32)
    pts = orc.occ_grid_points(V, 1.0, [0, 0, 0])
    sdf = (np.linalg.norm(pts.astype(np.float64), axis=1, keepdims=True) - 0.3).astype(np.float32)
    _, occ = orc.occ_update_with_sdf(sdf, None, 1.0, V, 512.0, 1e-4, 0, np.ones(V ** 3, np.float32), np.ones(V ** 3, np.uint8))
    grid = OccupancyGrid(V, 1.0, [0, 0, 0])
    grid.set_grid_occupancy(torch.from_numpy(occ).cuda())
    sph = Sphere(0.5, [0, 0, 0])
    to, td = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    _, te, _, tx, _ = sph.ray_intersection(to, td)
    rsp = grid.compute_samples_in_occupied_regions(to, td, te, tx, 2e-3, 32, False)
    exp = orc.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], o, d, te.cpu().numpy(), tx.cpu().numpy(), occ.astype(np.uint8), 2e-3, 32, False)
    assert np.array_equal(rsp.ray_start_end_idx.cpu().numpy(), exp.start_end), "ray sampling parity"

    # 3. one tiny training iteration (forward, losses, double backward, optimizer)
    hp = HyperParams()
    hp.max_nr_samples_per_ray = 16
    hp.nr_samples_imp_sampling = 4
    tr = Trainer(hp, nr_levels=4, capacity=2 ** 12, sdf_hidden=32, occupancy_resolution=64, with_colorcal=False, optimizer="fused")
    tr.set_analytic_scene()
    gt = torch.rand(256, 3, device="cuda"); gm = torch.ones(256, 1, device="cuda")
    before = tr.model_sdf.encoding.lattice_values.detach().clone()
    loss = tr.step(to, td, gt, gm, None, optimizer_step=False)
    lv = float(loss)
    assert np.isfinite(lv), "training step produced a non finite loss"
    gnorm = float(tr.model_sdf.encoding.lattice_values.grad.abs().sum())
    assert gnorm > 0, "no gradient reached the SDF lattice"
    tr.optimizer_step()                      # fused AdamW over the flat buffers (zeroes the gradients in the same pass)
    assert not torch.equal(before, tr.model_sdf.encoding.lattice_values.detach()), "the optimizer did not move the SDF lattice"
    if verbose:
        print("smoke ok: enc rel err %.2e, pos-grad rel err %.2e, %d samples, loss %.4f" % (e1, e2, tr.last["nr_samples"], lv))
    return True
