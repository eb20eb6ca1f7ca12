"""Sphere-tracing throughput (SURVEY.md 8d, config C5: one 1920x1080 frame of primary rays) with the fused single-kernel tracer
and with the reference-style masked Python loop on the same network. Prints one JSON line.
usage (under gpurun): python tools/bench_sphere_trace.py [--width 1920 --height 1080 --iters 30]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "compat")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--fit_iters", type=int, default=400)
    a = ap.parse_args()
    import permuto_sdf_b200.train as tr
    from permuto_sdf_b200.train import HyperParams, Trainer
    t = Trainer(HyperParams(), nr_levels=16, capacity=2 ** 18, sdf_hidden=64, nr_images=8, occupancy_resolution=256, seed=0, optimizer="fused")
    t.set_analytic_scene()
    m = t.model_sdf
    m.last_iter_nr = 20000
    # fit the SDF to the analytic sphere of the scene (the reference's sphere initialisation, train_permuto_sdf.py:262-291), so that
    # rays converge on a surface inside the occupied shell like they do on a trained model
    for i in range(a.fit_iters):
        loss, _, _ = tr.loss_sphere_init(30000, t.aabb, m, 20000)
        t.optimizer.zero_grad(set_to_none=False)
        loss.backward()
        t.optimizer_step()
    with torch.no_grad():
        chk = torch.nn.functional.normalize(torch.randn(4096, 3, device="cuda"), dim=-1) * 0.3
        fit_err = float(m(chk, 20000)[0].abs().mean())
    # pinhole camera at (0, 0, 1.5) looking at the origin
    W, H = a.width, a.height
    f = 1.2 * W
    u, v = torch.meshgrid(torch.arange(W, device="cuda", dtype=torch.float32), torch.arange(H, device="cuda", dtype=torch.float32), indexing="xy")
    # pixel centres (u + 0.5): no ray has an exactly zero direction component -- such rays creep by 1e-6 per DDA step in the reference's
    # marchers (SURVEY.md A.3, reproduced here) and would dominate the frame time
    d = torch.stack([(u + 0.5 - W / 2) / f, (v + 0.5 - H / 2) / f, torch.ones_like(u)], -1).reshape(-1, 3)
    d = torch.nn.functional.normalize(d, dim=-1).contiguous()
    o = torch.tensor([0.0, 0.0, -1.5], device="cuda").expand_as(d).contiguous()
    out = {}
    torch.set_grad_enabled(False)          # rendering: every network evaluation takes the fused tensor-core path
    tr.FUSED_SPHERE_TRACE_MAX_RAYS = 1 << 30          # compare both paths at every size
    for fused in (True, False):
        tr.FUSED_SPHERE_TRACE = fused
        for _ in range(2):
            pts, sdf, grads, geom, rsp = tr.sphere_trace(a.iters, o, d, m, True, 0.9, 1e-3, t.occupancy_grid)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.reps):
            pts, sdf, grads, geom, rsp = tr.sphere_trace(a.iters, o, d, m, True, 0.9, 1e-3, t.occupancy_grid)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / a.reps
        out["fused" if fused else "masked_loop"] = {"ms_per_frame": ms, "pixels_per_s": W * H / (ms / 1e3), "rays_hitting_grid": int(pts.shape[0])}
    tr.FUSED_SPHERE_TRACE = True
    print(json.dumps({"metric": "sphere-trace pixels/s (primary rays, %d iterations max, normals included)" % a.iters, "width": W, "height": H, "sdf_fit_mean_abs_error_on_surface": fit_err, **out}))


if __name__ == "__main__":
    main()
