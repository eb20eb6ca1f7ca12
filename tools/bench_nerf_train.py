"""NeRF training iteration at the reference shape (train_nerf.py: 512 rays, <= 64 foreground + 32 background samples per ray, 24 levels,
2^18 entries, deterministic mode) on the shaded-sphere scene of bench.py, with and without masks. Three paths, alternated over rounds:

    autograd   the loop of train_nerf.py: NerfHash (fused autograd) + VolumeRenderingNerf + torch losses + loss.backward() + torch AdamW
    eager      NerfTrainer's direct kernel sequence, launched eagerly
    graph      the same sequence replayed from captured CUDA graphs

Prints median ms per iteration (CUDA events over blocks of 8 iterations, so every block contains one occupancy refresh) and GPU operations
per iteration (kernels and memsets in a torch.profiler trace of 8 iterations), with the card's name and power limit, as one JSON line.

    python tools/bench_nerf_train.py [--rounds 5] [--iters 48]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit not read"


def make(kind, with_mask):
    from permuto_sdf_b200.graphs import graph_state
    from permuto_sdf_b200.nerf_train import NerfTrainer
    tr = NerfTrainer(8, with_mask, optimizer="adamw" if kind == "autograd" else "fused", deterministic=True, direct=(kind != "autograd"))
    if kind == "graph":
        graph_mode(True)
        tr._cg = graph_state(torch.cuda.Stream(), "occ", "step")       # enable_cuda_graph without the class-wide switch
    return tr


def draws(n_iter, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, H * W, (512,), generator=g).to(torch.int32).pin_memory(),
             torch.randint(0, 8, (512,), generator=g).to(torch.int32).pin_memory()) for _ in range(n_iter)]


def graph_mode(on):
    """the class-wide sampler state of graph replay (static-capacity containers, device-resident generators) for the graph path only: the
    autograd loop and the eager sequence run with exactly sized containers, as the reference does. The device generator tensors the
    graphs captured are kept and refilled, never replaced."""
    from permuto_sdf_b200.permuto_sdf import OccupancyGrid, RaySampler, RaySamplesPacked
    RaySamplesPacked.static_capacity = on
    sg = lambda v: v - (1 << 64) if v >= (1 << 63) else v
    for r in (OccupancyGrid.m_rng, RaySampler.m_rng):
        keep = getattr(r, "_bench_dev", None)
        if on and r.dev is None:
            if keep is None:
                r.to_device()
                r._bench_dev = r.dev
            else:
                keep.copy_(torch.tensor([sg(r.state), sg(r.inc)], dtype=torch.int64))
                r.dev = keep
        elif not on and r.dev is not None:
            r._bench_dev = r.dev
            r.to_host()


def run_block(tr, reel, d):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for pix, img in d:
        tr.step_from_reel(reel, pix, img)
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / len(d)


def ops_per_iter(tr, reel, d):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for pix, img in d:
            tr.step_from_reel(reel, pix, img)
        torch.cuda.synchronize()
    n = sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA)
    return n / len(d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=48, help="timed iterations per path and round (a multiple of 8)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nerf_train: needs a CUDA device")
    import bench
    H, W = 600, 800
    reel = bench.analytic_reel(8, H, W, 1000.0, torch.device("cuda"))
    result = {"card": card(), "shape": "512 rays, <=64+32 samples/ray, L24, T2^18, deterministic"}
    for with_mask in (False, True):
        paths = {}
        for kind in ("autograd", "eager", "graph"):
            graph_mode(kind == "graph")
            tr = make(kind, with_mask)
            for pix, img in draws(24, H, W, 1):                  # warm-up: iterations 0..23 (captures, the foreground window)
                tr.step_from_reel(reel, pix, img)
            torch.cuda.synchronize()
            paths[kind] = tr
        times = {k: [] for k in paths}
        for r in range(args.rounds):
            d = draws(args.iters, H, W, 100 + r)
            for kind, tr in paths.items():
                graph_mode(kind == "graph")
                for a in range(0, args.iters, 8):
                    times[kind].append(run_block(tr, reel, d[a:a + 8]))
        ops = {}
        for k, tr in paths.items():
            graph_mode(k == "graph")
            ops[k] = ops_per_iter(tr, reel, draws(8, H, W, 999))
        graph_mode(False)
        tag = "mask" if with_mask else "no_mask"
        result[tag] = {k: {"ms_per_iter_median": round(statistics.median(v), 4), "gpu_ops_per_iter": round(ops[k], 1)} for k, v in times.items()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
