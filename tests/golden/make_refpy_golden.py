"""Fixture generator: runs the reference's UNMODIFIED Python classes (permuto_sdf_py/models/models.py, volume_rendering/*.py,
utils/sdf_utils.py) on the CPU through oracle/refpy.py and stores seeded inputs, parameters, outputs and gradients in
tests/golden/refpy_golden.npz (+ refpy_golden_bg.npz). Needs a checkout of the original project, named by PERMUTO_SDF_REFERENCE; the GPU tests
(tests/test_refpy_golden_gpu.py) load the .npz, put the same parameters into the CUDA path and compare.

    python tests/golden/make_refpy_golden.py

The 24 x 2^18 x 2 hash tables are not stored: they are regenerated on both sides from `lattice_from_seed` (a torch CPU generator);
table gradients are stored sparsely (touched rows only).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def lattice_from_seed(seed, L, T, F, amp):
    g = torch.Generator().manual_seed(int(seed))
    return ((torch.rand(L, T, F, generator=g) * 2 - 1) * amp).contiguous()


def sparse_rows(grad):
    """[L,T,F] gradient -> (flat row indices int32, values [n,F]) of the touched rows"""
    g = grad.reshape(-1, grad.shape[-1])
    nz = (g != 0).any(dim=1).nonzero().view(-1)
    return nz.to(torch.int32).numpy(), g[nz].numpy()


def unit(x):
    return x / x.norm(dim=-1, keepdim=True)


def main():
    from oracle import refpy
    M = refpy.install()
    import permuto_sdf as ps                    # the CPU stand-ins installed above
    from permuto_sdf_py.utils import sdf_utils
    out = {}
    torch.manual_seed(1234)
    aabb = ps.Sphere(0.5, [0, 0, 0])
    L, T, F = 24, 2 ** 18, 2

    def put(prefix, sd):
        for k, v in sd.items():
            if "lattice_values" in k:
                continue
            out[prefix + k] = v.detach().cpu().numpy()

    # ------------------------------------------------------------------ SDF: value, gradient, curvature, parameter gradients
    sdf_m = M.SDF(in_channels=3, boundary_primitive=aabb, geom_feat_size_out=32, nr_iters_for_c2f=10000)
    with torch.no_grad():
        sdf_m.encoding.lattice_values.copy_(lattice_from_seed(11, L, T, F, 0.3))
        for p in sdf_m.mlp_sdf.parameters():                 # spread the biases so that the GELUs leave their linear regime
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.2)
    put("sdf.", sdf_m.state_dict())
    N = 192
    pts = unit(torch.randn(N, 3)) * torch.rand(N, 1) * 0.45
    it = 4000
    ca, cB, cC = torch.randn(N, 1), torch.randn(N, 3), torch.randn(N, 32)
    sdf, grad, geom = sdf_m.get_sdf_and_gradient(pts.clone(), it)
    loss = (sdf * ca).sum() + (grad * cB).sum() + (geom * cC).sum()
    sdf_m.zero_grad()
    loss.backward()
    out.update({"sdf_in.points": pts.numpy(), "sdf_in.iter": np.int64(it), "sdf_in.ca": ca.numpy(), "sdf_in.cB": cB.numpy(), "sdf_in.cC": cC.numpy(),
                "sdf_out.sdf": sdf.detach().numpy(), "sdf_out.grad": grad.detach().numpy(), "sdf_out.geom": geom.detach().numpy()})
    for k, p in sdf_m.named_parameters():
        if p.grad is None:
            continue
        if "lattice_values" in k:
            out["sdf_grad.lattice_rows"], out["sdf_grad.lattice_vals"] = sparse_rows(p.grad)
        else:
            out["sdf_grad." + k] = p.grad.numpy().copy()
    # curvature along a stored random direction (the reference draws it with torch.randn_like: patched for the call)
    rnd = torch.randn(N, 3)
    real_randn_like = torch.randn_like
    torch.randn_like = lambda t, *a, **k: rnd.clone()
    try:
        sdf_sh, curv = sdf_m.get_sdf_and_curvature_1d_precomputed_gradient_normal_based(pts.clone(), grad.detach(), it)
    finally:
        torch.randn_like = real_randn_like
    out.update({"curv_in.rnd": rnd.numpy(), "curv_out.sdf_shifted": sdf_sh.detach().numpy(), "curv_out.curvature": curv.detach().numpy()})

    # ------------------------------------------------------------------ RGB: Lipschitz MLP with active clamps + colour calibration
    rgb_m = M.RGB(in_channels=3, boundary_primitive=aabb, geom_feat_size_in=32, nr_iters_for_c2f=1)
    cal = M.Colorcal(4, 0)
    with torch.no_grad():
        rgb_m.encoding.lattice_values.copy_(lattice_from_seed(12, L, T, F, 0.3))
        for i, c in enumerate(rgb_m.mlp.lipshitz_bound_per_layer):
            c.mul_([0.35, 0.45, 1.0, 0.4][i])                 # softplus(c) below many row sums: the clamp is active
        cal.weight_delta.copy_(torch.randn(4, 3) * 0.1)
        cal.bias.copy_(torch.randn(4, 3) * 0.1)
    put("rgb.", rgb_m.state_dict())
    put("cal.", cal.state_dict())
    R = 24
    counts = torch.randint(0, 13, (R,))
    counts[3] = 0
    ends = torch.cumsum(counts, 0)
    se = torch.stack([ends - counts, ends], 1).to(torch.int32)
    Nr = int(ends[-1])
    rp = unit(torch.randn(Nr, 3)) * torch.rand(Nr, 1) * 0.45
    rd = unit(torch.randn(Nr, 3))
    rg = (torch.randn(Nr, 3) * torch.rand(Nr, 1) * 2).requires_grad_(True)
    rf = (torch.randn(Nr, 32) * 0.5).requires_grad_(True)
    img = torch.randint(0, 4, (R,), dtype=torch.int32)
    cw = torch.randn(Nr, 3)
    rgb = rgb_m(rp, rd, rg, rf, 20000, cal, img, se)
    rgb_m.zero_grad(); cal.zero_grad()
    (rgb * cw).sum().backward()
    out.update({"rgb_in.points": rp.numpy(), "rgb_in.dirs": rd.numpy(), "rgb_in.sdf_gradients": rg.detach().numpy(), "rgb_in.geom": rf.detach().numpy(),
                "rgb_in.img_indices": img.numpy(), "rgb_in.ray_start_end_idx": se.numpy(), "rgb_in.cw": cw.numpy(), "rgb_in.iter": np.int64(20000),
                "rgb_out.rgb": rgb.detach().numpy(), "rgb_grad.sdf_gradients": rg.grad.numpy().copy(), "rgb_grad.geom": rf.grad.numpy().copy()})
    seen = set()
    for k, p in list(rgb_m.named_parameters()) + [("cal." + k, p) for k, p in cal.named_parameters()]:
        if p.grad is None or id(p) in seen:
            continue
        seen.add(id(p))
        if "lattice_values" in k:
            out["rgb_grad.lattice_rows"], out["rgb_grad.lattice_vals"] = sparse_rows(p.grad)
        else:
            out["rgb_grad." + k] = p.grad.numpy().copy()

    # ------------------------------------------------------------------ background NeRF (4-D lattice)
    bg_m = M.NerfHash(4, boundary_primitive=aabb, nr_iters_for_c2f=1)
    with torch.no_grad():
        bg_m.encoding.lattice_values.copy_(lattice_from_seed(13, L, T, F, 0.3))
    put("bg.", bg_m.state_dict())
    Nb = 96
    bp = torch.cat([unit(torch.randn(Nb, 3)), torch.rand(Nb, 1)], 1)
    bd = unit(torch.randn(Nb, 3))
    cb, cd = torch.randn(Nb, 3), torch.randn(Nb, 1)
    brgb, bden = bg_m(bp, bd, 20000)
    bg_m.zero_grad()
    ((brgb * cb).sum() + (bden * cd).sum()).backward()
    out.update({"bg_in.points": bp.numpy(), "bg_in.dirs": bd.numpy(), "bg_in.cb": cb.numpy(), "bg_in.cd": cd.numpy(),
                "bg_out.rgb": brgb.detach().numpy(), "bg_out.density": bden.detach().numpy()})
    for k, p in bg_m.named_parameters():
        if p.grad is None:
            continue
        if "lattice_values" in k:
            out["bg_grad.lattice_rows"], out["bg_grad.lattice_vals"] = sparse_rows(p.grad)
        else:
            out["bg_grad." + k] = p.grad.numpy().copy()

    # ------------------------------------------------------------------ NeuS weights + integration on a ragged packed sample set
    rsp = ps.RaySamplesPacked(R, Nr)
    rsp.ray_start_end_idx = se.clone()
    rsp.samples_dirs = rd.clone()
    rsp.samples_dt = torch.rand(Nr, 1) * 0.01 + 1e-4
    rsp.samples_pos = rp.clone()
    ns = (torch.randn(Nr, 1) * 0.01).requires_grad_(True)
    ng = (unit(torch.randn(Nr, 3)) * (1 + 0.1 * torch.randn(Nr, 1))).requires_grad_(True)
    nrgb = torch.rand(Nr, 3).requires_grad_(True)
    cwt, cws, cpr = torch.randn(Nr, 1), torch.randn(R, 1), torch.randn(R, 3)
    for tag, forced in (("free", None), ("forced", 0.55)):
        for t in (ns, ng, nrgb):
            t.grad = None
        vr = M.VolumeRenderingNeus()          # a fresh module per mode (SingleVarianceNetwork re-registers last_variance as a Parameter)
        w, wsum, bgT, inv_s = vr.compute_weights(rsp, ns, ng, 0.4, forced)
        pred = vr.integrate(rsp, nrgb, w)
        ((w * cwt).sum() + (wsum * cws).sum() + (pred * cpr).sum() + (bgT * cws).sum() * 0.5).backward()
        out.update({"neus_%s.weights" % tag: w.detach().numpy(), "neus_%s.weights_sum" % tag: wsum.detach().numpy(),
                    "neus_%s.bg_transmittance" % tag: bgT.detach().numpy(), "neus_%s.inv_s" % tag: inv_s.detach().numpy().reshape(1),
                    "neus_%s.pred" % tag: pred.detach().numpy(), "neus_%s.g_sdf" % tag: ns.grad.numpy().copy(),
                    "neus_%s.g_gradients" % tag: ng.grad.numpy().copy(), "neus_%s.g_rgb" % tag: nrgb.grad.numpy().copy()})
        if forced is None:
            out["neus_free.g_variance"] = vr.deviation_network.variance.grad.numpy().reshape(1).copy()
    out.update({"neus_in.dt": rsp.samples_dt.numpy(), "neus_in.sdf": ns.detach().numpy(), "neus_in.gradients": ng.detach().numpy(),
                "neus_in.rgb": nrgb.detach().numpy(), "neus_in.cwt": cwt.numpy(), "neus_in.cws": cws.numpy(), "neus_in.cpr": cpr.numpy(),
                "neus_in.cos_anneal": np.float32(0.4), "neus_in.forced": np.float32(0.55)})

    # ------------------------------------------------------------------ drivers on an analytic SDF (identical arithmetic on CPU and GPU):
    # importance_sampling_sdf_model (sdf_utils.py:383-423) and sphere_trace (sdf_utils.py:120-218)
    class AnalyticSDF(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.boundary_primitive = aabb
            self.last_iter_nr = 0

        def forward(self, points, iter_nr):
            x, y, z = points[:, 0:1], points[:, 1:2], points[:, 2:3]
            return torch.sqrt(x * x + y * y + z * z) - 0.3, None

        def get_sdf_and_gradient(self, points, iter_nr):
            sdf, _ = self.forward(points, iter_nr)
            return sdf, points / (sdf + 0.3), None

    am = AnalyticSDF().eval()
    V = 64
    grid = ps.OccupancyGrid(V, 1.0, [0, 0, 0])
    centers = torch.from_numpy(refpy.ro.occ_grid_points(V, 1.0, np.zeros(3, np.float32)))
    occ = ((centers.norm(dim=1) - 0.3).abs() < 0.05)
    grid.set_grid_occupancy(occ)
    Rr = 96
    cam = unit(torch.randn(Rr, 3)) * 1.2
    tgt = torch.randn(Rr, 3) * 0.22
    ro_, rd_ = cam, unit(tgt - cam)
    _, te, _, tx, _ = aabb.ray_intersection(ro_, rd_)
    uni = grid.compute_samples_in_occupied_regions(ro_, rd_, te, tx, 1e-3, 40, False).compact_to_valid_samples()
    merged = sdf_utils.importance_sampling_sdf_model(am, uni, ro_, rd_, tx, 0)
    pts_t, sdf_t, grad_t, _, traced = sdf_utils.sphere_trace(30, ro_, rd_, am, True, 0.9, 1e-3, occupancy_grid=grid)
    out.update({"drv_in.origins": ro_.numpy(), "drv_in.dirs": rd_.numpy(), "drv_in.V": np.int64(V), "drv_in.occupancy": occ.numpy(),
                "imp_out.ray_start_end_idx": merged.ray_start_end_idx.numpy(), "imp_out.samples_z": merged.samples_z.numpy(),
                "imp_out.samples_pos": merged.samples_pos.numpy(), "imp_out.samples_dt": merged.samples_dt.numpy(),
                "trace_out.points": pts_t.numpy(), "trace_out.sdf": sdf_t.detach().numpy(),
                "trace_out.ray_start_end_idx": traced.ray_start_end_idx.numpy()})

    # two files, each under 1 MB: the background model's arrays (keys bg*) go to <name>_bg.npz
    path = os.environ.get("REFPY_GOLDEN_OUT") or os.path.join(ROOT, "tests", "golden", "refpy_golden.npz")
    np.savez_compressed(path, **{k: v for k, v in out.items() if not k.startswith("bg")})
    np.savez_compressed(path[:-len(".npz")] + "_bg.npz", **{k: v for k, v in out.items() if k.startswith("bg")})
    print("wrote %s (+ _bg): %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
