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

    python tools/bench_mesh.py [--res 512 1024 2000] [--rounds 3] [--ref-res 512]
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


def extract(model, N):
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    return extract_mesh_from_sdf_model(model, N, -0.5, 0.5)


def shares(model, N):
    """-> (seconds in the fused SDF forward, seconds in the marching-cubes entry points, wall seconds) of one instrumented extraction"""
    from permuto_sdf_b200 import _lib
    _lib.stats_begin(with_events=True)
    wall, _ = timed(lambda: extract(model, N))
    _, _, times = _lib.stats_end()
    ms = lambda names: sum(times.get(n, (0, 0.0))[1] for n in names) / 1e3
    return ms(["psdf_sdf_fused_forward"]), ms(["psdf_marching_cubes_count", "psdf_marching_cubes_emit"]), wall


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[512, 1024, 2000])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ref-res", type=int, default=512)
    a = ap.parse_args()
    gpu = card()
    model = fitted_model()
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
        print(json.dumps({"measure": "extract", "N": N, "seconds_median": statistics.median(times), "seconds": times,
                          "grid_points_per_s": N ** 3 / statistics.median(times),
                          "share_sdf_eval": t_eval / t_wall, "share_marching_cubes": t_mc / t_wall, "instrumented_seconds": t_wall,
                          "peak_alloc_MB": peak / 2 ** 20, "dense_volume_MB": N ** 3 * 4 / 2 ** 20, "vertices": nv, "faces": nf,
                          "card": gpu}), flush=True)
    if a.ref_res:
        N = a.ref_res
        reference_eval(model, 128)
        times = [reference_eval(model, N) for _ in range(a.rounds)]
        print(json.dumps({"measure": "ref_eval", "N": N, "seconds_median": statistics.median(times), "seconds": times,
                          "note": "evaluation stage only; the reference's skimage marching cubes is not measured", "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
