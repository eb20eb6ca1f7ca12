"""Time of one sphere-fit iteration (train_permuto_sdf.py:323-331: 30 000 points, SDF only) in three formulations, alternated in one run:

  loop          the hand-written autograd loop: loss_sphere_init + loss.backward() + Trainer.optimizer_step() (AdamW over every group)
  fit eager     Trainer.fit_sphere, the direct kernel sequence launched eagerly
  fit graph     Trainer.fit_sphere after enable_cuda_graph(): the same sequence replayed from one captured graph

16 levels, T = 2^18, 3 x 64 SDF MLP, deterministic mode. Times: CUDA events around `--iters` iterations, `--rounds` rounds per
formulation in turn, median over the rounds. Launches per iteration: CUDA kernels, memsets and copies in a torch.profiler trace of a
separate window. Prints one JSON line per formulation, with the card name and power limit.

    python tools/bench_sphere_fit.py [--iters 50] [--rounds 5]
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


def make(kind):
    import permuto_sdf_b200.train as T
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.nr_iter_sphere_fit = 1 << 30          # the timed windows never reach the end of the phase
    tr = Trainer(hp, nr_levels=16, capacity=2 ** 18, sdf_hidden=64, nr_images=8, occupancy_resolution=256, seed=0, optimizer="fused",
                 deterministic=True)
    if kind == "fit graph":
        tr.enable_cuda_graph()
    state = {"i": 0}

    def loop_iter():
        loss, _, _ = T.loss_sphere_init(30000, tr.aabb, tr.model_sdf, state["i"])
        tr.optimizer.zero_grad(set_to_none=False)
        loss.backward()
        tr.optimizer_step()
        state["i"] += 1

    def run(k):
        if kind == "loop":
            for _ in range(k):
                loop_iter()
        else:
            tr.fit_sphere(k)
    return tr, run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_sphere_fit.py needs a CUDA device")
    kinds = ("loop", "fit eager", "fit graph")
    runs = {k: make(k) for k in kinds}
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
    launches = {}
    n_prof = 10
    for k in kinds:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            runs[k][1](n_prof)
            torch.cuda.synchronize()
        dev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        launches[k] = len(dev) / n_prof
    c = card()
    for k in kinds:
        tr = runs[k][0]
        print(json.dumps(dict(variant=k, execution=tr.execution.get("sphere_fit") or "hand-written autograd loop",
                              ms_per_iter=round(statistics.median(ms[k]), 4), ms_per_iter_rounds=[round(x, 4) for x in ms[k]],
                              gpu_ops_per_iter=launches[k], iters=a.iters, rounds=a.rounds, card=c)), flush=True)
    for k in kinds:
        if runs[k][0]._cg is not None:
            runs[k][0].disable_cuda_graph()


if __name__ == "__main__":
    main()
