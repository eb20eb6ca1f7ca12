"""No-mask training step at the C2 shape: the autograd formulation with the per-op background NerfHash against the direct iteration
with the fused background (Trainer(fused_background=True)).

512 rays, 96 + 2 x 16 foreground and 32 background samples per ray, 16 levels, deterministic mode. Step time: CUDA events around
graph-replayed steps. Background call times: CUDA events around the library calls of the background in eager steps (per-op path:
the 4-D encoding kernels, whose MLP runs in torch and is not included; fused path: the fused forward, compositing and backward).
Prints one JSON line per configuration, with the card name and power limit.

    python tools/bench_background.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (scene helpers of the headline benchmark)

BG_CALLS = ("psdf_enc_forward", "psdf_enc_backward", "psdf_bg_fused_forward", "psdf_bg_fused_backward", "psdf_nerf_bg_composite_forward",
            "psdf_nerf_bg_composite_backward")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def run(fused, steps, warmup):
    from permuto_sdf_b200 import _lib
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.with_mask = False
    hp.max_nr_samples_per_ray = 96
    hp.nr_samples_imp_sampling = 16
    hp.nr_samples_bg = 32
    hp.nr_rays = 512
    tr = Trainer(hp, nr_levels=16, capacity=2 ** 18, sdf_hidden=64, nr_images=8, occupancy_resolution=256, seed=0, optimizer="fused",
                 deterministic=True, fused_background=fused, direct=None if fused else False)
    tr.set_analytic_scene()
    tr.iter_nr = 20000
    H, W, f = 600, 800, 1000.0
    reel = bench.analytic_reel(8, H, W, f, torch.device("cuda"))
    gen = torch.Generator().manual_seed(1000)
    total = steps + warmup
    pix = [bench.central_pixels(512, H, W, 300, gen).cuda() for _ in range(2 * total)]
    img = [torch.randint(0, 8, (512,), generator=gen, dtype=torch.int32).cuda() for _ in range(2 * total)]
    # eager steps: background call times
    for i in range(warmup):
        tr.step_from_reel(reel, pix[i], img[i], update_occupancy=(i % 8 == 0))
    torch.cuda.synchronize()
    _lib.stats_begin(with_events=True)
    for i in range(warmup, total):
        tr.step_from_reel(reel, pix[i], img[i], update_occupancy=(i % 8 == 0))
    _, _, times = _lib.stats_end()
    calls = {k: round(v[1] / steps, 4) for k, v in times.items() if k in BG_CALLS}
    # graph replay: step time
    tr.enable_cuda_graph(warmup_steps=3)
    for i in range(total, total + warmup):
        tr.step_from_reel(reel, pix[i], img[i], update_occupancy=(i % 8 == 0))
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(total + warmup, 2 * total):
        tr.step_from_reel(reel, pix[i], img[i], update_occupancy=(i % 8 == 0))
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / steps
    tr.disable_cuda_graph()
    return dict(config="direct iteration + fused background" if fused else "autograd formulation + per-op background",
                iteration=tr.execution["iteration"], background=tr.execution["background"], ms_per_step=round(ms, 4),
                background_call_ms_per_step=calls, card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_background.py needs a CUDA device")
    for fused in (False, True):
        print(json.dumps(run(fused, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
