"""Time of the connected-component calls of Mesh on meshes with many components of very different sizes.

Workload: the iso-surface at 0 of a synthetic field on the grid linspace(-0.5, 0.5, N)^3, meshed by the streamed marching-cubes kernels a
slab of slices at a time (mesh._mesh_grid, as extract_mesh_from_sdf_model does), so the N^3 volume never exists. The field is the minimum
of three distance fields:
  - one sphere of radius 0.3 at the origin;
  - blobs: the space is cut into cells of 1/20; a cell holds a sphere with probability 0.35, jittered in the cell, of radius 0.1-0.35
    of the cell (about 2500 outside the large sphere);
  - specks: cells of 1/160 hold a sphere of 0.3 cells with probability 0.002 (about 8000), each about one grid spacing at N = 512, so
    which of them are meshed and how finely depends on N.
Cell choices come from an integer hash of the cell index, so the volume is the same at every N and in every run.

Per N, after one warm-up of every call:
  connected_components       Mesh.connected_components(): the kernels, the read of the component count and the range check
  components_kernels         psdf_mesh_components alone (the five kernels)
  remove_small_components    Mesh.remove_small_components(100) on a copy of the mesh, compaction included
  keep_largest_component     Mesh.keep_largest_component() on a copy, compaction included
each the median over --rounds of CUDA events around the call (the calls end in a host read, so the events bracket finished work);
peak_alloc_MB is torch.cuda.max_memory_allocated during those calls above what the mesh and its copy hold. The CPU baseline (the project
this one was modelled on has no such step): the host copy of F a user would make, then scipy.sparse.csgraph.connected_components of the
vertex graph (the three edges of every face), median of --cpu-rounds wall times; skipped above --cpu-max-res. Prints one JSON line per N
with the card name and power limit read in the same run.

    python tools/bench_mesh_components.py [--res 512 1024 2000] [--rounds 5] [--cpu-rounds 3] [--cpu-max-res 2000]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat")]

from bench_mesh import card  # noqa: E402


def _hash01(ix, iy, iz, salt):
    """uniform [0, 1) from an integer cell index (int64 tensors)"""
    h = (ix * 73856093) ^ (iy * 19349663) ^ (iz * 83492791) ^ salt
    h = h & 0xFFFFFFFF
    h = (h * 2654435761) & 0xFFFFFFFF
    h = h ^ (h >> 15)
    h = (h * 2246822519) & 0xFFFFFFFF
    h = h ^ (h >> 13)
    return h.to(torch.float64).div_(2.0 ** 32).float()


def _cell_spheres(p, cell, prob, r_lo, r_hi, salt):
    """distance to the sphere of p's cell (1 where the cell has none)"""
    idx = torch.floor((p + 0.5) / cell).to(torch.int64)
    ix, iy, iz = idx.unbind(1)
    u = [_hash01(ix, iy, iz, salt + k) for k in range(5)]
    centre = (idx.float() + 0.5 + 0.3 * (torch.stack(u[:3], 1) - 0.5)) * cell - 0.5
    d = (p - centre).norm(dim=1) - cell * (r_lo + (r_hi - r_lo) * u[3])
    return torch.where(u[4] < prob, d, torch.ones_like(d))


def field(pts, out):
    d = pts.norm(dim=1) - 0.3
    d = torch.minimum(d, _cell_spheres(pts, 1.0 / 20, 0.35, 0.1, 0.35, 11))
    d = torch.minimum(d, _cell_spheres(pts, 1.0 / 160, 0.002, 0.3, 0.3, 101))
    out.copy_(d)


def make_mesh(N):
    from permuto_sdf_b200.mesh import Mesh, _mesh_grid
    with torch.no_grad():
        V, F = _mesh_grid(N, -0.5, 0.5, 0.0, torch.device("cuda"), field)
    return Mesh(V, F, torch.nn.functional.normalize(V, dim=1))


def copy(m):
    from permuto_sdf_b200.mesh import Mesh
    return Mesh(m.V.clone(), m.F.clone(), m.NV.clone())


def gpu_ms(fn, prepare=None, rounds=5):
    """median ms of CUDA events around fn(arg), arg = prepare() made outside the events"""
    out = []
    for _ in range(rounds):
        arg = prepare() if prepare else None
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn(arg)
        e.record()
        e.synchronize()
        out.append(s.elapsed_time(e))
        del arg
    return statistics.median(out), out


def scipy_seconds(m, rounds):
    import scipy.sparse
    import scipy.sparse.csgraph
    nv = m.V.shape[0]
    times, nr = [], None
    for _ in range(rounds):
        torch.cuda.synchronize()
        t = time.perf_counter()
        F = m.F.cpu().numpy()
        rows = np.concatenate([F[:, 0], F[:, 1], F[:, 2]])
        cols = np.concatenate([F[:, 1], F[:, 2], F[:, 0]])
        A = scipy.sparse.csr_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(nv, nv))
        nr, _ = scipy.sparse.csgraph.connected_components(A, directed=False)
        times.append(time.perf_counter() - t)
        del F, rows, cols, A
    return statistics.median(times), times, nr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[512, 1024, 2000])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cpu-rounds", type=int, default=3)
    ap.add_argument("--cpu-max-res", type=int, default=2000)
    a = ap.parse_args()
    from permuto_sdf_b200._lib import call, load_library
    gpu = card()
    for N in a.res:
        m = make_mesh(N)
        labels, nr, counts = m.connected_components(with_face_counts=True)
        sizes = counts[counts > 0]
        rec = {"measure": "mesh_components", "N": N, "vertices": m.V.shape[0], "faces": m.F.shape[0], "components": nr,
               "components_with_faces": int(sizes.numel()), "largest_faces": int(sizes.max()) if sizes.numel() else 0,
               "components_ge_100_faces": int((sizes >= 100).sum())}
        del labels, counts, sizes
        nv, nf = m.V.shape[0], m.F.shape[0]
        ws = torch.empty(int(load_library().psdf_mesh_components_workspace_bytes(nv, nf)), dtype=torch.uint8, device="cuda")
        runs = {"connected_components": (lambda _: m.connected_components(), None),
                "components_kernels": (lambda _: call("psdf_mesh_components", nv, nf, m.F, ws), None),
                "remove_small_components": (lambda c: c.remove_small_components(100), lambda: copy(m)),
                "keep_largest_component": (lambda c: c.keep_largest_component(), lambda: copy(m))}
        for fn, prep in runs.values():
            fn(prep() if prep else None)                                 # warm-up
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated() + m.V.nbytes + m.F.nbytes + m.NV.nbytes    # the mesh and the copy of it
        torch.cuda.reset_peak_memory_stats()
        for name, (fn, prep) in runs.items():
            med, all_ms = gpu_ms(fn, prep, a.rounds)
            rec[name + "_ms"] = med
            rec[name + "_ms_all"] = all_ms
        rec["peak_alloc_MB"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        kept = copy(m).remove_small_components(100)
        rec["after_remove_small_100"] = {"vertices": kept.V.shape[0], "faces": kept.F.shape[0]}
        kept = copy(m).keep_largest_component()
        rec["after_keep_largest"] = {"vertices": kept.V.shape[0], "faces": kept.F.shape[0]}
        del kept, ws
        if N <= a.cpu_max_res:
            s, all_s, nr_cpu = scipy_seconds(m, a.cpu_rounds)
            rec.update(scipy_with_copy_s=s, scipy_with_copy_s_all=all_s, scipy_components=nr_cpu)
            rec["speedup_vs_scipy"] = s * 1e3 / rec["connected_components_ms"]
        else:
            rec["scipy_with_copy_s"] = "not measured"
        rec["card"] = gpu
        print(json.dumps(rec), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
