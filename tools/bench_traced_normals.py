"""Time of the traced-normal display of the point-cloud and space-time programs in two formulations, alternated in one run:

  loop           the reference's sequence on the per-op kernels: AABB.ray_intersection, the masked gather / scatter loop of sphere_trace
                 (sdf_utils.py:120-218) evaluating SDF.forward, get_sdf_and_gradient under autograd at the end points,
                 filter_unconverged_points and F.normalize (the model with its fused paths switched off)
  trace_normals  SurfaceFit.trace_normals / SpaceTimeFit.trace_normals: the box intersection kernel, the fused tracer, one fused value +
                 gradient forward

Shapes: the frame of train_sdf_from_mesh.py:193 (500 x 500 rays, 20 iterations, multiplier 0.9, threshold 2e-4) and the one of
vis_4d_sdf.py:105 (800 x 510 rays, 40 iterations, multiplier 0.3, threshold 2e-3, time 0.4); 24 levels, T = 2^18, 3 x 32 SDF MLP. The
models are trained first (`--train` iterations of SurfaceFit on an off-centre sphere and of SpaceTimeFit on a moving sphere), so that the
rays converge as on a fitted model. Times: CUDA events around one frame, `--rounds` rounds per formulation in turn after a warm-up,
median over the rounds. Prints one JSON line per program with the card name and power limit read in the same run.

    python tools/bench_traced_normals.py [--rounds 7] [--train 1000]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def camera_rays(w, h, eye, look_at, fov_deg=40.0):
    eye, at = torch.tensor(eye, device="cuda"), torch.tensor(look_at, device="cuda")
    fwd = F.normalize(at - eye, dim=0)
    right = F.normalize(torch.linalg.cross(fwd, torch.tensor([0.0, 1.0, 0.0], device="cuda")), dim=0)
    up = torch.linalg.cross(right, fwd)
    tan = torch.tan(torch.tensor(fov_deg / 2 * 3.141592653589793 / 180))
    u = ((torch.arange(w, device="cuda").float() + 0.5) / w * 2 - 1) * tan
    v = ((torch.arange(h, device="cuda").float() + 0.5) / h * 2 - 1) * tan * h / w
    vv, uu = torch.meshgrid(v, u, indexing="ij")
    d = F.normalize(fwd + uu.reshape(-1, 1) * right + vv.reshape(-1, 1) * up, dim=1)
    return eye.expand_as(d).contiguous(), d.contiguous()


def per_op(fit, o, d, time_val, iters, mult, tresh):
    """the reference's sequence with the model's fused paths off"""
    from permuto_sdf_b200.train import filter_unconverged_points, sphere_trace
    m = fit.model_sdf
    saved = (m.fused, getattr(m, "fused_training", False), m.training, m.last_iter_nr)
    m.fused, m.fused_training = None, False
    m.eval()
    try:
        with torch.no_grad():
            m.last_iter_nr = fit.iter_nr - 1
            end, sdf, grad, _, _ = sphere_trace(iters, o, d, m, True, mult, tresh, None, time_val)
            _, grad_c, conv = filter_unconverged_points(end, sdf, grad)
            return end, F.normalize(grad, dim=1), F.normalize(grad_c, dim=1), conv
    finally:
        m.fused, m.fused_training = saved[0], saved[1]
        m.train(saved[2])
        m.last_iter_nr = saved[3]


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--train", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_traced_normals.py needs a CUDA device")
    from permuto_sdf_b200 import SpaceTimeFit, SurfaceFit
    gpu = card()
    g = torch.Generator(device="cuda").manual_seed(0)
    dirs = F.normalize(torch.randn(200000, 3, device="cuda", generator=g), dim=-1)
    c0 = torch.tensor([0.1, -0.05, 0.08], device="cuda")
    surf = SurfaceFit((c0 + 0.3 * dirs).contiguous(), dirs.contiguous())
    surf.enable_cuda_graph()
    surf.fit(args.train)
    frames, per = 221, 1000
    t = (torch.arange(frames, device="cuda").float() / (frames - 1)).repeat_interleave(per)
    d4 = F.normalize(torch.randn(t.shape[0], 3, device="cuda", generator=g), dim=-1)
    cen = torch.tensor([-0.15, 0.05, 0.0], device="cuda") + t[:, None] * torch.tensor([0.3, -0.1, 0.1], device="cuda")
    st = SpaceTimeFit(torch.cat([cen + (0.2 + 0.1 * t)[:, None] * d4, t[:, None]], 1).contiguous(), d4.contiguous())
    st.enable_cuda_graph()
    st.fit(args.train)
    torch.cuda.synchronize()
    progs = [("train_sdf_from_mesh.py:193", surf, camera_rays(500, 500, [0.1, 0.3, 1.4], [0.1, -0.05, 0.08]), None, 20, 0.9, 2e-4),
             ("vis_4d_sdf.py:105", st, camera_rays(800, 510, [0.0, 0.3, 1.4], [-0.03, 0.01, 0.04]), 0.4, 40, 0.3, 2e-3)]
    for name, fit, (o, d), time_val, iters, mult, tresh in progs:
        fused = (lambda: fit.trace_normals(o, d, iters, mult, tresh)) if time_val is None else \
            (lambda: fit.trace_normals(o, d, time_val, iters, mult, tresh))
        loop = lambda: per_op(fit, o, d, time_val, iters, mult, tresh)
        for fn in (loop, fused):           # warm-up: modules, allocator, cuBLAS handles
            timed(fn)
        times = {"loop": [], "trace_normals": []}
        outs = {}
        for _ in range(args.rounds):
            for k, fn in (("loop", loop), ("trace_normals", fused)):
                ms, outs[k] = timed(fn)
                times[k].append(ms)
        a, b = outs["loop"], outs["trace_normals"]
        both = (a[3] * b[3]).view(-1) > 0
        res = {"program": name, "rays": int(o.shape[0]), "iterations": iters, "multiplier": mult, "threshold": tresh, "time_val": time_val,
               "ms_median": {k: statistics.median(v) for k, v in times.items()}, "ms_all": times,
               "speedup": statistics.median(times["loop"]) / statistics.median(times["trace_normals"]),
               "converged": {"loop": int(a[3].sum()), "trace_normals": int(b[3].sum()), "differ": int((a[3] != b[3]).sum())},
               "max_normal_diff_where_both_converged": float((a[1] - b[1]).abs().max(dim=1).values[both].max()) if bool(both.any()) else None,
               "card": gpu, "rounds": args.rounds, "train_iterations": args.train}
        print(json.dumps(res))


if __name__ == "__main__":
    main()
