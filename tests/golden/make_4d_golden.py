"""Fixture generator for the space-time SDF: runs the reference's UNMODIFIED SDF(in_channels=4, ...) (permuto_sdf_py/models/models.py),
AABB (utils/aabb.py) and sdf_loss (utils/sdf_utils.py) on the CPU through oracle/refpy.py, as one iteration of train_4d_sdf.py:200-237 on
seeded points, and stores the inputs, the model state, sdf, the [N,4] gradient of get_sdf_and_gradient, the loss and every parameter
gradient in tests/golden/refpy_golden_4d.npz. Needs a checkout of the original project, named by PERMUTO_SDF_REFERENCE;
tests/test_spacetime_fit_gpu.py loads the .npz and compares SpaceTimeFit's direct sequence and its per-op fallback.

    python tests/golden/make_4d_golden.py

The rows are those SpaceTimeFit forms from its draws: the Ns sequence rows (here the whole sequence, in order), then the box rows of
aabb.rand_points_inside from the stored uniform draw u01 and the time column ut. The hash table is regenerated from a seed on both
sides (make_refpy_golden.lattice_from_seed); its gradient is stored sparsely.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_refpy_golden import lattice_from_seed, sparse_rows, unit  # noqa: E402

L, T, F = 24, 2 ** 18, 2
SEED = 31
ITER = 1500                      # the coarse-to-fine window of nr_iters_for_c2f = 3000 in mid-ramp
NS, NO = 192, 160


def main():
    from oracle import refpy
    M = refpy.install()
    from permuto_sdf_py.utils.aabb import AABB
    from permuto_sdf_py.utils.sdf_utils import sdf_loss
    torch.manual_seed(4242)
    aabb = AABB(bounding_box_sizes_xyz=[1.0, 1.0, 1.0], bounding_box_translation=[0.0, 0.0, 0.0])
    m = M.SDF(in_channels=4, boundary_primitive=aabb, geom_feat_size_out=0, nr_iters_for_c2f=3000)
    with torch.no_grad():
        m.encoding.lattice_values.copy_(lattice_from_seed(SEED, L, T, F, 0.3))
        for p in m.mlp_sdf.parameters():                  # spread the biases so that the GELUs leave their linear regime
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.2)
    out = {"state." + k: v.detach().numpy().copy() for k, v in m.state_dict().items() if "lattice_values" not in k}
    # the sequence rows (a moving sphere, times in [0, 1]) and the box rows of train_4d_sdf.py:205-207
    g = torch.Generator().manual_seed(7)
    t = torch.rand(NS, 1, generator=g)
    d = unit(torch.randn(NS, 3, generator=g))
    cloud = torch.cat([d * (0.2 + 0.1 * t) + t * torch.tensor([0.3, -0.1, 0.1]), t], 1)
    normals = d.clone()
    torch.manual_seed(99)
    u01 = torch.rand(NO, 3)
    torch.manual_seed(99)
    box = aabb.rand_points_inside(nr_points=NO)              # the same draw: u01 * size - size / 2 + translation
    ut = torch.rand((NO, 1))
    points_time = torch.cat([cloud, torch.cat([box, ut], 1)], 0)
    sdf, sdf_gradients_time, _ = m.get_sdf_and_gradient(points_time, ITER)
    sdf_gradients = sdf_gradients_time[:, 0:3]
    loss = sdf_loss(sdf[:NS], sdf_gradients[:NS], sdf[-NO:], sdf_gradients[-NO:], normals) / 30000
    m.zero_grad()
    loss.backward()
    out.update({"in.cloud": cloud.numpy(), "in.normals": normals.numpy(), "in.u01": u01.numpy(), "in.ut": ut.numpy(),
                "in.iter": np.int64(ITER), "in.seed": np.int64(SEED), "out.points_time": points_time.detach().numpy(),
                "out.sdf": sdf.detach().numpy(), "out.grad4": sdf_gradients_time.detach().numpy(),
                "out.loss": loss.detach().numpy().reshape(1)})
    for k, p in m.named_parameters():
        if p.grad is None:
            continue
        if "lattice_values" in k:
            out["grad.lattice_rows"], out["grad.lattice_vals"] = sparse_rows(p.grad)
        else:
            out["grad." + k] = p.grad.numpy().copy()
    path = os.environ.get("GOLDEN_4D_OUT") or os.path.join(ROOT, "tests", "golden", "refpy_golden_4d.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
