"""Fixture generator for sphere tracing with an AABB boundary: runs the reference's UNMODIFIED AABB (permuto_sdf_py/utils/aabb.py),
SDF (models/models.py), sphere_trace and filter_unconverged_points (utils/sdf_utils.py) on the CPU through oracle/refpy.py and stores
tests/golden/refpy_golden_trace.npz. Needs a checkout of the original project, named by PERMUTO_SDF_REFERENCE;
tests/test_traced_normals_gpu.py loads the .npz and compares AABB.ray_intersection, SurfaceFit.trace_normals and
SpaceTimeFit.trace_normals.

    python tests/golden/make_trace_golden.py

Cases (the parameters of the programs' display blocks):
  "d3"    SDF(3, AABB, 0, 5000), sphere_trace(20, ..., sdf_multiplier=0.9, sdf_converged_tresh=2e-4)   train_sdf_from_mesh.py:193
  "d4_a"  SDF(in_channels=4, AABB, 0, 3000), the same call with sdf_multiplier=0.7 and time_val 0.25  train_4d_sdf.py:268
  "d4_b"  the same model at time_val 0.8
The boxes are non-cubic and translated. The rays include misses, origins inside the box and axis-parallel directions (with origins on a
box face, whose slab test divides 0 by 0). Hash tables come from a seed on both sides (make_refpy_golden.lattice_from_seed with
amplitude 1, times a per-level amplitude 0.3 * 0.5^l that is stored: a smooth field), the MLP weights are stored. The output layer is
scaled so that the median |d sdf / dx| in the box is 1 and shifted so that the median sdf there is 0: an SDF-like field on which a fair
share of the rays converges.

The stand-in RaySamplesPacked of oracle/refpy.py lacks initialize_with_one_sample_per_ray (src/RaySamplesPacked.cu:97-120), which
sphere_trace calls without an occupancy grid; it is added here as that C++ method reads.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_refpy_golden import lattice_from_seed, unit  # noqa: E402

L, T, F = 24, 2 ** 18, 2
ITERS = {"d3": 5000, "d4": 3000}                 # the windows are fully open (nr_iters_for_c2f of each program)
SEEDS = {"d3": 41, "d4": 43}
BOXES = {"d3": ([0.9, 1.1, 0.8], [0.05, -0.1, 0.02]), "d4": ([1.2, 0.9, 1.0], [-0.05, 0.04, 0.1])}
CASES = [("d3", "d3", None, 0.9, 2e-4, 20), ("d4_a", "d4", 0.25, 0.7, 2e-4, 20), ("d4_b", "d4", 0.8, 0.7, 2e-4, 20)]
RAY_SEEDS = {"d3": 11, "d4_a": 12, "d4_b": 13}
N_RAYS = {"d3": 1536, "d4": 768}
LEVEL_AMP = (0.3 * 0.5 ** torch.arange(L, dtype=torch.float64)).float()


def _init_one_sample_per_ray(self, one_sample_per_ray, dirs):
    n = one_sample_per_ray.shape[0]
    self.samples_pos, self.samples_dirs = one_sample_per_ray, dirs
    self.samples_z, self.samples_dt, self.ray_fixed_dt = torch.zeros(n, 1), torch.zeros(n, 1), torch.zeros(n, 1)
    idx = torch.arange(n).view(-1, 1)
    self.ray_start_end_idx = torch.cat([idx, idx + 1], 1)
    self.cur_nr_samples = torch.tensor([n], dtype=torch.int32)
    self.rays_have_equal_nr_of_samples, self.fixed_nr_of_samples_per_ray = True, 1


def make_rays(n, size, trans, g):
    """rays at the box: 60 % from outside towards a point inside, 15 % from outside away from it (misses), 15 % from inside the box,
    10 % with one or two direction components exactly 0, some of them starting on a box face"""
    size, trans = torch.tensor(size), torch.tensor(trans)
    n_in, n_away, n_axis = int(0.15 * n), int(0.15 * n), int(0.10 * n)
    n_to = n - n_in - n_away - n_axis
    far = lambda k: trans + unit(torch.randn(k, 3, generator=g)) * (1.2 + 0.6 * torch.rand(k, 1, generator=g))
    inside = lambda k: trans + (torch.rand(k, 3, generator=g) - 0.5) * size * 0.9
    o_to = far(n_to)
    d_to = unit(inside(n_to) - o_to)
    o_away = far(n_away)
    d_away = unit(o_away - trans + 0.3 * torch.randn(n_away, 3, generator=g))
    o_in = inside(n_in)
    d_in = unit(torch.randn(n_in, 3, generator=g))
    o_ax = inside(n_axis) + (torch.rand(n_axis, 3, generator=g) - 0.5) * size * 0.8
    d_ax = torch.randn(n_axis, 3, generator=g)
    for i in range(n_axis):
        zero = [i % 3] if i % 2 == 0 else [i % 3, (i + 1) % 3]
        d_ax[i, zero] = 0.0
        if i % 5 == 0:                             # on the face of a zeroed axis: (bb - o) / 0 = 0 / 0
            k = zero[0]
            o_ax[i, k] = float(-size[k] / 2 + trans[k]) if i % 10 == 0 else float(size[k] - size[k] / 2 + trans[k])
    d_ax = unit(d_ax)
    o = torch.cat([o_to, o_away, o_in, o_ax], 0).float().contiguous()
    d = torch.cat([d_to, d_away, d_in, d_ax], 0).float().contiguous()
    return o, d


def main():
    from oracle import refpy
    M = refpy.install()
    import permuto_sdf as ps
    ps.RaySamplesPacked.initialize_with_one_sample_per_ray = _init_one_sample_per_ray
    from permuto_sdf_py.utils.aabb import AABB
    from permuto_sdf_py.utils.sdf_utils import filter_unconverged_points, sphere_trace
    out = {}
    models = {}
    for key, D, c2f in (("d3", 3, 5000), ("d4", 4, 3000)):
        torch.manual_seed(SEEDS[key])
        size, trans = BOXES[key]
        aabb = AABB(bounding_box_sizes_xyz=size, bounding_box_translation=trans)
        m = M.SDF(in_channels=D, boundary_primitive=aabb, geom_feat_size_out=0, nr_iters_for_c2f=c2f)
        with torch.no_grad():
            m.encoding.lattice_values.copy_(lattice_from_seed(SEEDS[key], L, T, F, 1.0) * LEVEL_AMP.view(L, 1, 1))
        # output layer: median gradient norm 1 and median sdf 0 over uniform space-time points of the box
        g = torch.Generator().manual_seed(SEEDS[key] + 1)
        lo_hi = [(t - s / 2, s) for s, t in zip(size, trans)] + ([(0.0, 1.0)] if D == 4 else [])
        probe = torch.rand(4000, D, generator=g) * torch.tensor([w for _, w in lo_hi]) + torch.tensor([a for a, _ in lo_hi])
        s_p, g_p, _ = m.get_sdf_and_gradient(probe, ITERS[key])
        c, med = 1.0 / float(g_p[:, :3].detach().norm(dim=1).median()), float(s_p.detach().median())
        with torch.no_grad():
            m.mlp_sdf[-1].weight.mul_(c)
            m.mlp_sdf[-1].bias.sub_(med).mul_(c)
        m.eval()
        models[key] = m
        out.update({key + ".state." + k: v.detach().numpy().copy() for k, v in m.state_dict().items() if "lattice_values" not in k})
        out.update({key + ".seed": np.int64(SEEDS[key]), key + ".iter": np.int64(ITERS[key]), key + ".box_size": np.float64(size),
                    key + ".box_translation": np.float64(trans), key + ".level_amp": LEVEL_AMP.numpy()})
    for name, key, time_val, mult, tresh, n_iters in CASES:
        m = models[key]
        g = torch.Generator().manual_seed(RAY_SEEDS[name])
        o, d = make_rays(N_RAYS[key], *BOXES[key], g)
        pe, te, px, tx, hit = m.boundary_primitive.ray_intersection(o, d)
        m.last_iter_nr = ITERS[key]
        with torch.no_grad():
            pts, sdf, grad, _, _ = sphere_trace(n_iters, o, d, m, return_gradients=True, sdf_multiplier=mult, sdf_converged_tresh=tresh,
                                                time_val=time_val)
        _, grad_conv, is_conv = filter_unconverged_points(pts, sdf, grad)
        p = name + "."
        out.update({p + "origins": o.numpy(), p + "dirs": d.numpy(), p + "pts_entry": pe.numpy(), p + "t_entry": te.numpy(),
                    p + "pts_exit": px.numpy(), p + "t_exit": tx.numpy(), p + "hit": hit.numpy(), p + "ray_end": pts.detach().numpy(),
                    p + "sdf": sdf.detach().numpy(), p + "grad": grad.detach().numpy(), p + "is_converged": is_conv.detach().numpy(),
                    p + "time_val": np.float64(-1.0 if time_val is None else time_val), p + "mult": np.float64(mult),
                    p + "tresh": np.float64(tresh), p + "nr_iters": np.int64(n_iters)})
        near = (sdf.abs() < tresh).float().mean()
        print("%s: %d rays, %d hit the box, converged (|sdf| < %g) %.3f, is_converged (sdf < 0.01) %.3f"
              % (name, o.shape[0], int(hit.sum()), tresh, float(near), float(is_conv.mean())))
    path = os.environ.get("GOLDEN_TRACE_OUT") or os.path.join(ROOT, "tests", "golden", "refpy_golden_trace.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
