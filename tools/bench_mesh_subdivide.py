"""Time of Mesh.upsample and Mesh.load on extracted meshes.

Workload: the mesh extract_mesh_from_sdf_model makes of the SDF of Trainer after fit_sphere() (bench_mesh.py's model, radius 0.3) on
linspace(-0.5, 0.5, N)^3, reduced to its largest component, as bench_mesh_decimate.py does. Per mesh:
  upsample   1 and 2 rounds of midpoint (smooth=False) and Loop (smooth=True) subdivision of a copy of the mesh, NV None: the median over
             --rounds of CUDA events around the call after one warm-up (the call reads the edge count from the device every round, so
             the events bracket finished work), the faces and vertices it makes, and peak_alloc_MB, torch.cuda.max_memory_allocated
             during the call above what was allocated before it;
  oracle     (--oracle-res only) one round of each mode by oracle/subdivide.py, the numpy restatement, on the host (wall clock, one run):
             it is the bit-exact reference, not a tuned CPU implementation, and says nothing about libigl, which is not measured;
  load       Mesh.load of the mesh saved as binary PLY (save_to_file) and as binary STL (welded, the default), from a temporary
             directory: the median wall time over --rounds of load to the GPU, ending in a device synchronise.
Prints one JSON line per mesh with the card name and power limit read in the same run.

    python tools/bench_mesh_subdivide.py [--res 512 1024] [--rounds 3] [--oracle-res 512]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tools")]

from bench_mesh import card, fitted_model  # noqa: E402
from bench_mesh_decimate import copy, events_ms  # noqa: E402


def upsample_stats(m, n, smooth, rounds):
    ms = []
    copy(m).upsample(n, smooth)                           # warm-up
    for _ in range(rounds):
        c = copy(m)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t, _ = events_ms(lambda: c.upsample(n, smooth))
        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        ms.append(t)
        faces, verts = c.F.shape[0], c.V.shape[0]
        del c
    return {"rounds": n, "smooth": smooth, "faces": faces, "vertices": verts, "ms": statistics.median(ms), "ms_all": ms,
            "peak_alloc_MB": round(peak, 1)}


def load_stats(m, rounds):
    from permuto_sdf_b200.mesh import Mesh
    out = {}
    with tempfile.TemporaryDirectory() as d:
        ply, stl = os.path.join(d, "m.ply"), os.path.join(d, "m.stl")
        m.save_to_file(ply)
        tri = m.V.cpu().numpy()[m.F.long().cpu().numpy()]
        rec = np.zeros(len(tri), dtype=[("n", "<f4", (3,)), ("v", "<f4", (3, 3)), ("attr", "<u2")])
        rec["v"] = tri
        with open(stl, "wb") as f:
            f.write(b"bench".ljust(80, b" ") + np.uint32(len(tri)).tobytes() + rec.tobytes())
        for name, p in (("ply", ply), ("stl", stl)):
            ts = []
            for _ in range(rounds + 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = Mesh.load(p)
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            out[name] = {"bytes": os.path.getsize(p), "ms": statistics.median(ts[1:]), "ms_all": ts[1:], "vertices": r.V.shape[0],
                         "faces": r.F.shape[0]}
            del r
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--res", type=int, nargs="*", default=[512, 1024])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--oracle-res", type=int, nargs="*", default=[512])
    args = ap.parse_args()
    from oracle import subdivide as S
    from permuto_sdf_b200 import extract_mesh_from_sdf_model
    gpu = card()
    model = fitted_model()
    for N in args.res:
        m = extract_mesh_from_sdf_model(model, N, -0.5, 0.5).keep_largest_component()
        m.NV = None
        rec = {"mesh": "sphere", "N": N, "vertices": m.V.shape[0], "faces": m.F.shape[0], "gpu": gpu}
        rec["upsample"] = [upsample_stats(m, n, smooth, args.rounds) for smooth in (False, True) for n in (1, 2)]
        if N in args.oracle_res:
            V, Fc = m.V.cpu().numpy(), m.F.cpu().numpy()
            rec["oracle_host_numpy"] = []
            for smooth in (False, True):
                t0 = time.perf_counter()
                S.upsample(V, Fc, 1, smooth)
                rec["oracle_host_numpy"].append({"rounds": 1, "smooth": smooth, "ms": (time.perf_counter() - t0) * 1e3})
        rec["load"] = load_stats(m, args.rounds)
        print(json.dumps(rec), flush=True)
        del m


if __name__ == "__main__":
    main()
