"""Per-kernel timings on the GPU (CUDA events, warm, median of reps): our kernels, and the reference's own
kernels (oracle/_ref) on the same inputs where available. Writes gpurun_out/microbench.json.
usage: python tools/microbench.py [--rays 512] [--samples 128] [--levels 16]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "compat")]
import scenes  # noqa: E402
from oracle import ref_gpu  # noqa: E402
from permuto_sdf_b200 import call  # noqa: E402


def timeit(fn, reps=30, warm=5, flush=None):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=512)
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--levels", type=int, default=16)
    ap.add_argument("--capacity", type=int, default=2 ** 18)
    a = ap.parse_args()
    import permutohedral_encoding as pe
    from permuto_sdf import OccupancyGrid, Sphere, VolumeRendering as VR
    res = {}
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 3350.0}
    hbm = peaks["hbm_gbs"]
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
    N, L, T = a.rays * a.samples, a.levels, a.capacity
    torch.manual_seed(0)
    enc = pe.PermutoEncoding(3, T, L, 2, np.geomspace(1.0, 1e-4, L), concat_points=True, concat_points_scaling=1e-3)
    # positions: samples along rays through the shell (spatially coherent like the real workload)
    o, d = scenes.make_rays(a.rays, seed=0, miss_fraction=0.0, axis_aligned=0)
    z = np.linspace(0.75, 1.0, a.samples, dtype=np.float32)
    pos = (o[:, None, :] + z[None, :, None] * d[:, None, :]).reshape(-1, 3).astype(np.float32)
    pos_t = torch.from_numpy(pos).cuda()
    rand_t = (torch.rand(N, 3, device="cuda") - 0.5)
    C = enc.output_dims()
    win = torch.ones(L, device="cuda")
    g_out = torch.randn(N, C, device="cuda")
    gg = torch.randn(N, 3, device="cuda")
    out = torch.empty(N, C, device="cuda")
    g_l = torch.zeros_like(enc.lattice_values)
    g_p = torch.empty(N, 3, device="cuda")
    g_go = torch.empty(N, C, device="cuda")
    lat = enc.lattice_values.detach()
    D = 3

    def args(p):
        return (N, D, L, 2, T, p, lat, enc.scale_factor, enc.shift_tensor(), win, 1, 1e-3)
    for name, p in (("ray", pos_t), ("rand", rand_t)):
        for fl, tag in ((None, "warm"), (flush, "coldL2")):
            med, mn = timeit(lambda: call("psdf_enc_forward", *args(p), out), flush=fl)
            res["enc_fwd_%s_%s" % (name, tag)] = dict(us=med, us_min=mn, GBs=N * (12 + L * 4 * 8 + C * 4) / med / 1e3)
            med, mn = timeit(lambda: call("psdf_enc_backward", *args(p), g_out, g_l, None), flush=fl)
            res["enc_bwd_lattice_%s_%s" % (name, tag)] = dict(us=med, us_min=mn, GBs=N * (12 + L * 8 + L * 4 * 8) / med / 1e3)
            med, mn = timeit(lambda: call("psdf_enc_backward", *args(p), g_out, None, g_p), flush=fl)
            res["enc_bwd_pos_%s_%s" % (name, tag)] = dict(us=med, us_min=mn)
            med, mn = timeit(lambda: call("psdf_enc_backward", *args(p), g_out, g_l, g_p), flush=fl)
            res["enc_bwd_both_%s_%s" % (name, tag)] = dict(us=med, us_min=mn)
            med, mn = timeit(lambda: call("psdf_enc_double_backward", *args(p), gg, g_out, g_l, g_go), flush=fl)
            res["enc_dbl_bwd_%s_%s" % (name, tag)] = dict(us=med, us_min=mn)
    med, mn = timeit(lambda: g_l.zero_())
    res["zero_lattice_grad"] = dict(us=med, GBs=g_l.numel() * 4 / med / 1e3)
    # torch MLP at this size (cuBLAS fp32) for comparison with the fused kernel later
    mlp = torch.nn.Sequential(torch.nn.Linear(C, 64), torch.nn.GELU(), torch.nn.Linear(64, 64), torch.nn.GELU(), torch.nn.Linear(64, 64),
                              torch.nn.GELU(), torch.nn.Linear(64, 33)).cuda()
    with torch.no_grad():
        med, mn = timeit(lambda: mlp(out))
    res["torch_mlp_fwd_64"] = dict(us=med)
    # ray ops: ours vs the reference kernels
    V = 256
    grid = OccupancyGrid(V, 1.0, [0, 0, 0])
    pts = grid.compute_grid_points(False)
    grid.update_with_sdf((pts.norm(dim=1, keepdim=True) - 0.3).contiguous(), 512.0, 1e10, 1e-4)
    sph = Sphere(0.5, [0, 0, 0])
    to, td = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    pe_, te, px, tx, hit = sph.ray_intersection(to, td)
    med, _ = timeit(lambda: sph.ray_intersection(to, td)); res["sphere_intersection"] = dict(us=med)
    med, _ = timeit(lambda: grid.compute_samples_in_occupied_regions(to, td, te, tx, 1e-4, 96, True)); res["occ_samples_api"] = dict(us=med)
    rsp = grid.compute_samples_in_occupied_regions(to, td, te, tx, 1e-4, 96, True)
    med, _ = timeit(lambda: rsp.compact_to_valid_samples()); res["compact_api"] = dict(us=med)
    c = rsp.compact_to_valid_samples()
    Ns = c.samples_pos.shape[0]
    res["nr_samples"] = Ns
    w = torch.rand(Ns, 1, device="cuda"); rgb = torch.rand(Ns, 3, device="cuda"); al = torch.rand(Ns, 1, device="cuda") * .2 + .8
    for nm, fn in (("cumprod", lambda: VR.cumprod_alpha2transmittance(c, al)), ("integrate", lambda: VR.integrate_with_weights(c, rgb, w)),
                   ("sum1", lambda: VR.sum_over_each_ray(c, w)), ("cdf", lambda: VR.compute_cdf(c, w)),
                   ("sdf2alpha", lambda: VR.sdf2alpha(c, w, 512, True, 1.0))):
        med, _ = timeit(fn); res["vr_%s_api" % nm] = dict(us=med)
    if ref_gpu.available():
        occ = grid.get_grid_occupancy()
        med, _ = timeit(lambda: ref_gpu.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], to, td, te, tx, occ, 1e-4, 96, True))
        res["REF_occ_samples"] = dict(us=med)
        rp = ref_gpu.Packed(a.rays, Ns)
        rp.pos, rp.dirs, rp.z, rp.dt, rp.fixed_dt, rp.start_end = c.samples_pos, c.samples_dirs, c.samples_z, c.samples_dt, c.ray_fixed_dt, c.ray_start_end_idx
        rp.max_nr_samples = Ns
        for nm, fn in (("cumprod", lambda: ref_gpu.vr_cumprod(rp, al)), ("integrate", lambda: ref_gpu.vr_integrate(rp, rgb, w)),
                       ("sum1", lambda: ref_gpu.vr_sum(rp, w)), ("cdf", lambda: ref_gpu.vr_cdf(rp, w)),
                       ("sdf2alpha", lambda: ref_gpu.vr_sdf2alpha(rp, w, 512, True, 1.0))):
            med, _ = timeit(fn); res["REF_vr_%s" % nm] = dict(us=med)
    res["hbm_peak_gbs"] = hbm
    od = os.path.join(ROOT, "gpurun_out"); os.makedirs(od, exist_ok=True)
    json.dump(res, open(os.path.join(od, "microbench.json"), "w"), indent=1)
    for k, v in res.items():
        print(k, v)


if __name__ == "__main__":
    main()
