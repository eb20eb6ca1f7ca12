"""Time of Mesh.decimate on extracted meshes, to 10 % and 1 % of their faces.

Workloads:
  sphere   the mesh extract_mesh_from_sdf_model makes of the SDF of Trainer after fit_sphere() (bench_mesh.py's model, radius 0.3) on
           linspace(-0.5, 0.5, N)^3, reduced to its largest component (the fitted network has crossings of its own towards the corners);
  blobs    the many-component field of bench_mesh_components.py (a sphere, about 2500 blobs and 8000 specks), as extracted.
Per mesh and target, after one warm-up call: the median over --rounds of CUDA events around Mesh.decimate on a copy of the mesh (the
call reads a count from the device every round, so the events bracket finished work), the number of rounds, the faces reached, and
peak_alloc_MB, torch.cuda.max_memory_allocated during the call above what the mesh and its copy hold. For the sphere the extraction itself
(extract_mesh_from_sdf_model, median of --rounds) is timed in the same run for comparison. Prints one JSON line per mesh with the card
name and power limit read in the same run.

    python tools/bench_mesh_decimate.py [--sphere-res 512 1024 2000] [--blobs-res 512 1024] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tools")]

from bench_mesh import card, fitted_model  # noqa: E402
from bench_mesh_components import make_mesh  # noqa: E402


def copy(m):
    from permuto_sdf_b200.mesh import Mesh
    return Mesh(m.V.clone(), m.F.clone(), None if m.NV is None else m.NV.clone())


def events_ms(fn):
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e), out


def decimate_stats(m, target, rounds):
    ms = []
    copy(m).decimate(target)                              # warm-up
    for _ in range(rounds):
        c = copy(m)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t, _ = events_ms(lambda: c.decimate(target))
        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        ms.append(t)
        faces = c.F.shape[0]
        del c
    nr = copy(m)._decimate(target)[3]
    return {"target": target, "faces": faces, "rounds": nr, "ms": statistics.median(ms), "ms_all": ms, "peak_alloc_MB": round(peak, 1)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--sphere-res", type=int, nargs="*", default=[512, 1024, 2000])
    ap.add_argument("--blobs-res", type=int, nargs="*", default=[512, 1024])
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    gpu = card()
    model = fitted_model() if args.sphere_res else None
    meshes = []
    for N in args.sphere_res:
        extract_mesh_from_sdf_model(model, N, -0.5, 0.5)
        ext = [events_ms(lambda: extract_mesh_from_sdf_model(model, N, -0.5, 0.5)) for _ in range(args.rounds)]
        mesh = ext[-1][1].keep_largest_component()
        meshes.append(("sphere", N, mesh, statistics.median(t for t, _ in ext)))
        del ext
    for N in args.blobs_res:
        meshes.append(("blobs", N, make_mesh(N), None))
    for kind, N, m, extract_ms in meshes:
        nf = m.F.shape[0]
        rec = {"mesh": kind, "N": N, "vertices": m.V.shape[0], "faces": nf, "gpu": gpu}
        if extract_ms is not None:
            rec["extract_ms"] = extract_ms
        rec["decimate"] = [decimate_stats(m, int(frac * nf), args.rounds) for frac in (0.1, 0.01)]
        print(json.dumps(rec), flush=True)
        del m


if __name__ == "__main__":
    main()
