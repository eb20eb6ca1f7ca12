"""Time of the image metrics (metrics.psnr / metrics.ssim, csrc/image_metrics.cu) and of Trainer.evaluate.

Workloads:
  kernels    psnr + ssim of B = 1 and 16 random [B,3,H,W] images with a mask and quantize_x, at 1200 x 1600 (DTU, pooled by 5), 576 x 768
             (by 2) and 2048 x 2048 (by 8), against the same metrics written the way piq writes them (fp32 torch: the quantization and the
             mask, the squared-difference mean, F.avg_pool2d and a grouped F.conv2d with the 11 x 11 window, then the formulas). The two
             alternate in one process: per round, CUDA events around --iters calls of each; the median, min and max over --rounds.
  evaluate   Trainer.evaluate of one 1200 x 1600 frame (bench.py's analytic reel, Trainer after fit_sphere): the wall time of the call,
             split into render_frame (ending in a device synchronise) and the metrics on its rows (CUDA events), median over --rounds.
Prints one JSON line with the card name and power limit read in the same run.

    python tools/bench_image_metrics.py [--rounds 5] [--iters 20]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tools")]

from bench_mesh import card  # noqa: E402
from permuto_sdf_b200 import metrics  # noqa: E402


def piq_style(x, y, m):
    """psnr and ssim as piq computes them (fp32), after the 8-bit round trip of x and the mask"""
    x = torch.clamp(torch.round(x * 255), 0, 255) / 255 * m
    y = y * m
    p = -10 * torch.log10(torch.mean((x - y) ** 2, dim=[1, 2, 3]) + 1e-8)
    f = max(1, round(min(x.size()[-2:]) / 256))
    if f > 1:
        x, y = F.avg_pool2d(x, kernel_size=f), F.avg_pool2d(y, kernel_size=f)
    c = torch.arange(11, dtype=x.dtype, device=x.device) - 5.0
    g = (-(c[None, :] ** 2 + c[:, None] ** 2) / (2 * 1.5 ** 2)).exp()
    g = (g / g.sum()).expand(x.size(1), 1, 11, 11)
    conv = lambda a: F.conv2d(a, g, groups=x.size(1))
    mx, my = conv(x), conv(y)
    sxx, syy, sxy = conv(x * x) - mx * mx, conv(y * y) - my * my, conv(x * y) - mx * my
    cs = (2 * sxy + 0.03 ** 2) / (sxx + syy + 0.03 ** 2)
    ss = (2 * mx * my + 0.01 ** 2) / (mx * mx + my * my + 0.01 ** 2) * cs
    return p, ss.mean(dim=(-1, -2)).mean(1)


def ours(x, y, m):
    return metrics.psnr(x, y, m[:, 0], True), metrics.ssim(x, y, m[:, 0], True)


def timed(fn, iters):
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def spread(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def kernels(rounds, iters):
    out = {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for H, W in ((1200, 1600), (576, 768), (2048, 2048)):
        for B in (1, 16):
            x = torch.rand(B, 3, H, W, device="cuda", generator=g)
            y = torch.rand(B, 3, H, W, device="cuda", generator=g)
            m = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.3).float()
            a, b = ours(x, y, m), piq_style(x, y, m)                 # warm-up of both
            t = {"ours": [], "piq_style_fp32": []}
            for _ in range(rounds):
                t["ours"].append(timed(lambda: ours(x, y, m), iters))
                t["piq_style_fp32"].append(timed(lambda: piq_style(x, y, m), iters))
            out["%dx%d_B%d" % (H, W, B)] = {"pool": metrics.pool_factor(H, W), "ms_per_call": {k: spread(v) for k, v in t.items()},
                                            "max_abs_diff_psnr_dB": float((a[0] - b[0].double()).abs().max()),
                                            "max_abs_diff_ssim": float((a[1] - b[1].double()).abs().max())}
    return out


def evaluate(rounds):
    import bench
    from permuto_sdf_b200.train import HyperParams, Trainer
    tr = Trainer(HyperParams(), seed=5, optimizer="fused")
    tr.set_analytic_scene()
    tr.fit_sphere()
    reel = bench.analytic_reel(1, 1200, 1600, 1400.0, torch.device("cuda"))
    tr.evaluate(reel)                                               # warm-up
    total, render, metric = [], [], []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = tr.evaluate(reel)
        total.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rgb = tr.render_frame(reel, 0)[0]
        torch.cuda.synchronize()
        render.append((time.perf_counter() - t0) * 1e3)
        y, m = reel.rgb_reel[0:1], reel.mask_reel[0]
        metric.append(timed(lambda: (metrics.psnr(rgb, y, m, True), metrics.ssim(rgb, y, m, True)), 1))
    return {"frame": "1200x1600", "ms_evaluate": spread(total), "ms_render_frame": spread(render), "ms_metrics": spread(metric),
            "psnr": res["psnr_mean"], "ssim": res["ssim_mean"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    res = {"card": card(), "kernels": kernels(a.rounds, a.iters), "evaluate": evaluate(a.rounds)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
