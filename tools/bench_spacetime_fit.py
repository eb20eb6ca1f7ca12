"""Time of one space-time SDF iteration (train_4d_sdf.py:194-241: 3000 sequence points + 3000 box points with a time column) in three
formulations, alternated in one run:

  loop          the reference's autograd loop: index_select + box and time draws, SDF(4).get_sdf_and_gradient on the per-op kernels,
                [:, :3], sdf_loss / 30000, loss.backward(), torch.optim.AdamW (SpaceTimeFit(optimizer="adamw"), whose step() is that loop)
  fit eager     SpaceTimeFit.step(), the direct kernel sequence launched eagerly
  fit graph     SpaceTimeFit.step() after enable_cuda_graph(): the same sequence replayed from one captured graph

The reference's shape: 24 levels, T = 2^18, 3 x 32 SDF MLP, out_dim 1; deterministic mode; a sequence of 221 frames of a moving sphere,
1000 points each.
Times: CUDA events around `--iters` iterations, `--rounds` rounds per formulation in turn, median over the rounds. GPU operations per
iteration: CUDA kernels, memsets and copies in a torch.profiler trace of a separate window. Prints one JSON line per formulation, with
the card name and power limit.

    python tools/bench_spacetime_fit.py [--iters 50] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def cloud(per_frame=1000, frames=221):
    g = torch.Generator(device="cuda").manual_seed(0)
    t = (torch.arange(frames, device="cuda").float() / (frames - 1)).repeat_interleave(per_frame)
    d = torch.nn.functional.normalize(torch.randn(t.shape[0], 3, device="cuda", generator=g), dim=-1)
    c = torch.tensor([-0.15, 0.05, 0.0], device="cuda") + t[:, None] * torch.tensor([0.3, -0.1, 0.1], device="cuda")
    r = 0.2 + 0.1 * t[:, None]
    return torch.cat([c + r * d, t[:, None]], 1).contiguous(), d.contiguous()


def make(kind, pts, nrm):
    from permuto_sdf_b200 import SpaceTimeFit
    fit = SpaceTimeFit(pts, nrm, optimizer="adamw" if kind == "loop" else "fused", deterministic=True)
    if kind == "fit graph":
        fit.enable_cuda_graph()

    def run(k):
        for _ in range(k):
            fit.step()
    return fit, run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_spacetime_fit.py needs a CUDA device")
    pts, nrm = cloud()
    kinds = ("loop", "fit eager", "fit graph")
    runs = {k: make(k, pts, nrm) for k in kinds}
    for k in kinds:                                  # warm-up: every shape, the graph capture
        runs[k][1](5)
    torch.cuda.synchronize()
    ms = {k: [] for k in kinds}
    for _ in range(a.rounds):
        for k in kinds:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            runs[k][1](a.iters)
            e.record()
            torch.cuda.synchronize()
            ms[k].append(s.elapsed_time(e) / a.iters)
    ops = {}
    n_prof = 10
    for k in kinds:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            runs[k][1](n_prof)
            torch.cuda.synchronize()
        dev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        ops[k] = len(dev) / n_prof
    c = card()
    for k in kinds:
        fit = runs[k][0]
        print(json.dumps(dict(variant=k, execution=fit.execution["step"], ms_per_iter=round(statistics.median(ms[k]), 4),
                              ms_per_iter_rounds=[round(x, 4) for x in ms[k]], gpu_ops_per_iter=ops[k], iters=a.iters, rounds=a.rounds,
                              card=c)), flush=True)
    for k in kinds:
        runs[k][0].disable_cuda_graph()


if __name__ == "__main__":
    main()
