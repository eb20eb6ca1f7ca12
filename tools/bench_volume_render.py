"""Time of one volume-rendered frame (the renderer of the reference's PSNR, orbit and novel-view images, train_permuto_sdf.py:172-209) in
two formulations, alternated in one run:

  run_net_in_chunks   per-op SDF encoder + autograd gradient, per-op compositing, chunks of 3000 rays (create_my_images.py:80)
  Trainer.render      the fused kernel sequence of permuto_sdf_b200/render.py at its default chunk

Scene as `bench.py --workload sphere_trace`: 16 levels, T = 2^18, 3 x 64 SDF MLP fitted to the analytic sphere (400 iterations), then the
whole occupancy grid refreshed from the fitted SDF so that sample counts are those of a fitted model; camera at z = -1.5 looking along +z,
focal length 1.2 W. Models in eval() (no jitter), iteration 20000, cos_anneal_ratio 1, forced variance hp.forced_variance_finish. Times:
host clock around a frame ending in a device synchronise (both paths sync on the host at every compaction), `--rounds` rounds per path
in turn after one warm-up frame each, median. Prints one JSON line with the card name and power limit, ms/frame and px/s per path, samples
per frame, the top C-ABI entry points per path (CUDA events, separate frame) and the largest |difference| between the two images.

    python tools/bench_volume_render.py [--width 800 --height 800] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def scene():
    import permuto_sdf_b200.train as T
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    tr = Trainer(hp, nr_levels=16, capacity=2 ** 18, sdf_hidden=64, nr_images=8, occupancy_resolution=256, seed=0, optimizer="fused",
                 deterministic=True)
    tr.set_analytic_scene()
    m = tr.model_sdf
    for _ in range(400):                      # the sphere fit of bench.py --workload sphere_trace
        loss, _, _ = T.loss_sphere_init(30000, tr.aabb, m, 20000)
        tr.optimizer.zero_grad(set_to_none=False)
        loss.backward()
        tr.optimizer_step()
    m.eval(); tr.model_rgb.eval()
    with torch.no_grad():                     # occupancy of the fitted SDF over the whole grid
        g = tr.occupancy_grid
        sdf, _, _ = m.fused(g.compute_grid_points(False), 20000, with_gradient=False, with_geom=False)
        g.update_with_sdf(sdf.contiguous(), 512.0, 1e10, 1e-4)
    return tr


def rays(W, H, dev):
    f, cx, cy = 1.2 * W, W / 2.0, H / 2.0
    v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
    d = torch.stack([(u + 0.5 - cx) / f, (v + 0.5 - cy) / f, torch.ones_like(u)], -1).reshape(-1, 3)
    d = torch.nn.functional.normalize(d, dim=-1).contiguous()
    o = torch.tensor([0.0, 0.0, -1.5], device=dev).expand_as(d).contiguous()
    return o, d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=800)
    ap.add_argument("--height", type=int, default=800)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_volume_render.py needs a CUDA device")
    from permuto_sdf_b200 import _lib
    from permuto_sdf_b200.render import DEFAULT_CHUNK
    from permuto_sdf_b200.train import run_net_in_chunks
    tr = scene()
    hp = tr.hp
    o, d = rays(a.width, a.height, torch.device("cuda"))
    it, cos, fv = 20000, 1.0, hp.forced_variance_finish
    paths = {
        "run_net_in_chunks": lambda: run_net_in_chunks(o, d, 3000, hp.with_mask, hp, tr.model_sdf, tr.model_rgb, tr.model_bg,
                                                       tr.occupancy_grid, it, cos, fv),
        "Trainer.render": lambda: tr.render(o, d, DEFAULT_CHUNK, it, cos, fv),
    }
    imgs = {k: f() for k, f in paths.items()}         # warm-up frame of each path
    torch.cuda.synchronize()
    ms = {k: [] for k in paths}
    for _ in range(a.rounds):
        for k, f in paths.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            imgs[k] = f()
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1e3)
    top, samples = {}, None
    for k, f in paths.items():                         # per entry point CUDA-event times, a separate frame
        _lib.stats_begin(with_events=True)
        f()
        _, launches, times = _lib.stats_end()
        if k == "Trainer.render":
            samples = _lib.LAST_UNITS.get("psdf_rgb_fused_forward", 0)       # composited samples (after importance resampling)
        top[k] = {"c_abi_launches": launches,
                  "top5_ms": {n: round(t, 3) for t, n in sorted(((v[1], n) for n, v in times.items()), reverse=True)[:5]}}
    px = a.width * a.height
    res = {}
    for k in paths:
        med = statistics.median(ms[k])
        res[k] = {"ms_per_frame": round(med, 3), "ms_rounds": [round(x, 3) for x in ms[k]], "px_per_s": round(px / (med / 1e3)),
                  **top[k]}
    diff = {name: float((x - y).abs().max()) for name, x, y in zip(("rgb", "normals", "weights_sum"),
                                                                  (imgs["Trainer.render"][i] for i in (0, 2, 3)),
                                                                  (imgs["run_net_in_chunks"][i] for i in (0, 2, 3)))}
    print(json.dumps(dict(frame="%dx%d" % (a.width, a.height), card=card(), samples_per_frame=samples, chunk={"run_net_in_chunks": 3000,
                          "Trainer.render": DEFAULT_CHUNK}, rounds=a.rounds, paths=res,
                          speedup=round(res["run_net_in_chunks"]["ms_per_frame"] / res["Trainer.render"]["ms_per_frame"], 3),
                          max_abs_diff=diff)), flush=True)


if __name__ == "__main__":
    main()
