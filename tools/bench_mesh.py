"""Time of mesh extraction from a trained SDF (extract_mesh_from_sdf_model) at the resolutions the reference's evaluation programs use.

  extract     permuto_sdf_b200.extract_mesh_from_sdf_model: the grid evaluated by the fused forward a slab of slices at a time, streamed
              through the marching-cubes kernels, then the fused value + gradient forward at the vertices for the normals
  ref_eval    the evaluation stage of the reference's extract_mesh_from_sdf_model (sdf_utils.py:260-277) restated: 64^3 chunks through the
              per-op SDF.forward (the model's fused paths switched off), each chunk copied with .cpu() into a dense float32 numpy array
              of N^3 values. Its marching-cubes stage (skimage, CPU) is not run here and not estimated.

The model is the SDF of Trainer after fit_sphere() (the sphere-fit phase of train_permuto_sdf.py, radius 0.3; reference sizes: 24 levels,
T = 2^18, 3 x 32 MLP). Per resolution N: the median wall time over `--rounds` extractions (host clock around work that ends in a device
synchronise), after one warm-up extraction; the shares of the fused SDF evaluation (grid and normals) and of the marching-cubes kernels,
from CUDA events around their entry points in one more, instrumented extraction; the peak device memory of an extraction
(torch.cuda.max_memory_allocated, above what was allocated before it) against the N^3 x 4 B dense volume; the vertex and face counts.
Prints one JSON line per measurement with the card name and power limit read in the same run.

--model nerf: the same for extract_mesh_from_density_model on the foreground NerfHash of a NerfTrainer (reference sizes: 24 levels,
T = 2^18) trained with masks on bench.analytic_reel (the shaded sphere of radius 0.3), at --threshold. ref_eval is then the evaluation
stage of the reference's extract_mesh_from_density_model (sdf_utils.py:341-366) restated: 64^3 chunks through the per-op
NerfHash.get_only_density, .cpu() into a dense numpy array. One more line, `density_kernel`, times the density-only kernel
(psdf_nerf_density_forward) against the full forward whose colour it discards (psdf_nerf_fused_forward at D = 3) at one slab of the grid
(2^24 points) and at the 65 536 points of NerfTrainer's occupancy refresh: CUDA events around --kernel-reps launches of each, the two
alternated over the rounds, median per launch.

    python tools/bench_mesh.py [--res 512 1024 2000] [--rounds 3] [--ref-res 512]
    python tools/bench_mesh.py --model nerf [--res 512 1024] [--iters 1500] [--threshold 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat")]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def fitted_model():
    from permuto_sdf_b200.train import HyperParams, Trainer
    tr = Trainer(HyperParams(), seed=5, optimizer="fused")
    tr.set_analytic_scene()
    tr.fit_sphere()
    torch.cuda.synchronize()
    return tr.model_sdf


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def trained_nerf(iters):
    """NerfTrainer (24 levels, T = 2^18) with masks, `iters` iterations on the analytic reel -> its foreground NerfHash(3)"""
    import bench
    from permuto_sdf_b200.nerf_train import NerfTrainer
    reel = bench.analytic_reel(9, 60, 80, 100.0, torch.device("cuda"))
    tr = NerfTrainer(9, True)
    g = torch.Generator().manual_seed(5)
    for _ in range(iters):
        pix = torch.randint(0, 60 * 80, (512,), generator=g).to(torch.int32)
        img = torch.randint(0, 8, (512,), generator=g).to(torch.int32)
        tr.step_from_reel(reel, pix, img)
    torch.cuda.synchronize()
    return tr.model


KIND = {"sdf": ("extract_mesh_from_sdf_model", "psdf_sdf_fused_forward"),
        "nerf": ("extract_mesh_from_density_model", "psdf_nerf_density_forward")}
ARGS = {"kind": "sdf", "threshold": 0.0}


def extract(model, N):
    import permuto_sdf_b200
    return getattr(permuto_sdf_b200, KIND[ARGS["kind"]][0])(model, N, -0.5, 0.5, threshold=ARGS["threshold"])


def shares(model, N):
    """-> (seconds in the fused forward, seconds in the marching-cubes entry points, wall seconds) of one instrumented extraction"""
    from permuto_sdf_b200 import _lib
    _lib.stats_begin(with_events=True)
    wall, _ = timed(lambda: extract(model, N))
    _, _, times = _lib.stats_end()
    ms = lambda names: sum(times.get(n, (0, 0.0))[1] for n in names) / 1e3
    return ms([KIND[ARGS["kind"]][1]]), ms(["psdf_marching_cubes_count", "psdf_marching_cubes_emit"]), wall


def reference_eval(model, N):
    """sdf_utils.py:260-277 on the per-op model: -> seconds"""
    saved = model.fused, getattr(model, "fused_training", False)
    model.fused, model.fused_training = None, False
    try:
        def run():
            with torch.no_grad():
                lin = torch.linspace(-0.5, 0.5, N, device="cuda")
                X = Y = Z = lin.split(64)
                sdf_full = np.zeros([N, N, N], dtype=np.float32)
                for xi, xs in enumerate(X):
                    for yi, ys in enumerate(Y):
                        for zi, zs in enumerate(Z):
                            xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing="ij")
                            pts = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1)
                            sdf_cur, _ = model(pts, 9999999)
                            sdf_full[xi * 64: xi * 64 + len(xs), yi * 64: yi * 64 + len(ys), zi * 64: zi * 64 + len(zs)] = \
                                sdf_cur.reshape(len(xs), len(ys), len(zs)).cpu().numpy()
                return sdf_full
        return timed(run)[0]
    finally:
        model.fused, model.fused_training = saved


def reference_density_eval(model, N):
    """sdf_utils.py:341-366 on the per-op NerfHash.get_only_density: -> seconds"""
    saved, model.fused = model.fused, None
    try:
        def run():
            with torch.no_grad():
                X = Y = Z = torch.linspace(-0.5, 0.5, N, device="cuda").split(64)
                full = np.zeros([N, N, N], dtype=np.float32)
                for xi, xs in enumerate(X):
                    for yi, ys in enumerate(Y):
                        for zi, zs in enumerate(Z):
                            xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing="ij")
                            pts = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1)
                            cur = model.get_only_density(pts, 9999999)
                            full[xi * 64: xi * 64 + len(xs), yi * 64: yi * 64 + len(ys), zi * 64: zi * 64 + len(zs)] = \
                                cur.reshape(len(xs), len(ys), len(zs)).cpu().numpy()
                return full
        return timed(run)[0]
    finally:
        model.fused = saved


def density_kernels(model, n, reps, rounds):
    """-> (ms per launch of the density-only kernel, of the full forward) at n points: medians over `rounds` alternated windows"""
    from permuto_sdf_b200._lib import call
    fb, enc = model.fused, model.encoding
    fb.pack(fb.params())
    g = torch.Generator(device="cuda").manual_seed(1)
    pts = torch.rand(n, 3, device="cuda", generator=g) - 0.5
    dirs = torch.zeros(n, 3, device="cuda")
    rgb, den = torch.empty(n, 3, device="cuda"), torch.empty(n, 1, device="cuda")
    e = (enc.nr_levels, enc.capacity)
    tail = (enc.scale_factor, enc.shift_tensor(), fb._window(9999999), enc.concat_points_scaling, fb.blob)
    lat = enc.lattice_values.detach()
    runs = {"density": lambda: call("psdf_nerf_density_forward", n, *e, pts, lat, *tail, den),
            "full": lambda: call("psdf_nerf_fused_forward", 3, n, *e, pts, dirs, lat, *tail, rgb, den)}
    out = {k: [] for k in runs}
    for k in runs:
        runs[k]()
    for _ in range(rounds):
        for k, fn in runs.items():
            s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(reps):
                fn()
            t.record()
            t.synchronize()
            out[k].append(s.elapsed_time(t) / reps)
    return statistics.median(out["density"]), statistics.median(out["full"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ref-res", type=int, default=512)
    ap.add_argument("--model", choices=("sdf", "nerf"), default="sdf")
    ap.add_argument("--iters", type=int, default=1500, help="--model nerf: training iterations")
    ap.add_argument("--threshold", type=float, default=None, help="iso-level (default: 0 for sdf, 20 for nerf)")
    ap.add_argument("--kernel-reps", type=int, default=20)
    a = ap.parse_args()
    nerf = a.model == "nerf"
    if a.res is None:
        a.res = [512, 1024] if nerf else [512, 1024, 2000]
    ARGS["kind"] = a.model
    ARGS["threshold"] = a.threshold if a.threshold is not None else (20.0 if nerf else 0.0)
    gpu = card()
    model = trained_nerf(a.iters) if nerf else fitted_model()
    extract(model, 256)
    for N in a.res:
        extract(model, N)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        times, mesh = [], None
        for _ in range(a.rounds):
            mesh = None
            t, mesh = timed(lambda: extract(model, N))
            times.append(t)
        peak = torch.cuda.max_memory_allocated() - base
        nv, nf = mesh.V.shape[0], mesh.F.shape[0]
        del mesh
        t_eval, t_mc, t_wall = shares(model, N)
        rec = {"measure": "extract", "N": N, "seconds_median": statistics.median(times), "seconds": times,
               "grid_points_per_s": N ** 3 / statistics.median(times),
               "share_density_eval" if nerf else "share_sdf_eval": t_eval / t_wall, "share_marching_cubes": t_mc / t_wall,
               "instrumented_seconds": t_wall, "peak_alloc_MB": peak / 2 ** 20, "dense_volume_MB": N ** 3 * 4 / 2 ** 20, "vertices": nv,
               "faces": nf, "card": gpu}
        if nerf:
            rec.update(model="nerf", threshold=ARGS["threshold"])
        print(json.dumps(rec), flush=True)
    if a.ref_res:
        N = a.ref_res
        ref = reference_density_eval if nerf else reference_eval
        ref(model, 128)
        times = [ref(model, N) for _ in range(a.rounds)]
        rec = {"measure": "ref_eval", "N": N, "seconds_median": statistics.median(times), "seconds": times,
               "note": "evaluation stage only; the reference's skimage marching cubes is not measured", "card": gpu}
        if nerf:
            rec["model"] = "nerf"
        print(json.dumps(rec), flush=True)
    if nerf:
        for n in (1 << 24, 65536):
            d, f = density_kernels(model, n, a.kernel_reps, max(a.rounds, 5))
            print(json.dumps({"measure": "density_kernel", "points": n, "density_only_ms": d, "full_forward_ms": f, "speedup": f / d,
                              "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
