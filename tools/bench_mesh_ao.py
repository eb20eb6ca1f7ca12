"""Time of the BVH build, Mesh.ambient_occlusion and load_mesh_sequence.

Workload:
  bvh / ao   sphere-in-sphere meshes (marching cubes of the union of two concentric spheres of radii 0.42 N and 0.15 N cells on an N^3
             grid, N chosen for about --faces faces): psdf_mesh_bvh_build and psdf_mesh_ambient_occlusion (S = 100) on a preallocated
             workspace, each the median over --rounds of CUDA events around the call after one warm-up, and the rays per second of the
             latter (V S rays);
  sequence   13 frames of a moving sphere-in-sphere of about 17 k faces each (about 270 k after two Loop rounds), written as OBJ to a
             temporary directory: load_mesh_sequence end to end (wall clock ending in a device synchronise, median over --rounds after a
             warm-up), and the same steps one at a time, each ending in a synchronise: load, normalise, normals + 2 Loop rounds, ambient
             occlusion of frame 0, vertex removal, interpolation + normals, concatenation.
Prints one JSON line per record with the card name and power limit read in the same run.

    python tools/bench_mesh_ao.py [--faces 300000 1000000 4000000] [--rounds 5]
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

from bench_mesh import card  # noqa: E402
from bench_mesh_decimate import events_ms  # noqa: E402


def spheres(N):
    from permuto_sdf_b200.mesh import marching_cubes
    c = (N - 1) / 2 + 0.31
    ax = torch.arange(N, device="cuda", dtype=torch.float32) - c
    r = torch.sqrt(ax[:, None, None] ** 2 + ax[None, :, None] ** 2 + ax[None, None, :] ** 2)
    V0, F0 = marching_cubes(r - 0.42 * N)                       # two closed spheres, each wound outward
    V1, F1 = marching_cubes(r - 0.15 * N)
    del r
    # rotated out of the grid planes: a ray in a plane of marching-cubes vertices meets shared edges exactly, where the fp32 test may pass neither face
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(11), dtype=torch.float64))
    V = (torch.cat([V0, V1]).double() / N) @ q.t().cuda()
    return V.float().contiguous(), torch.cat([F0, F1 + V0.shape[0]])


def grid_for(target):
    _, F = spheres(64)
    return max(16, int(round(64 * (target / F.shape[0]) ** 0.5)))


def bvh_ao(target, rounds, S=100):
    from permuto_sdf_b200._lib import call, load_library
    from permuto_sdf_b200.mesh import Mesh, fibonacci_directions
    N = grid_for(target)
    V, Fc = spheres(N)
    m = Mesh(V, Fc).recalculate_normals()
    nv, nf = V.shape[0], Fc.shape[0]
    ws = torch.empty(int(load_library().psdf_mesh_bvh_workspace_bytes(nv, nf)), dtype=torch.uint8, device="cuda")
    dirs = torch.from_numpy(fibonacci_directions(S)).cuda()
    vis = torch.empty(nv, device="cuda")
    build = lambda: call("psdf_mesh_bvh_build", nv, nf, V, Fc, ws)
    ao = lambda: call("psdf_mesh_ambient_occlusion", nv, nf, S, V, m.NV, dirs, ws, vis)
    build()
    ao()
    tb = [events_ms(build)[0] for _ in range(rounds)]
    ta = [events_ms(ao)[0] for _ in range(rounds)]
    assert torch.equal(vis, m.ambient_occlusion(S))
    ms_ao = statistics.median(ta)
    return {"N": N, "vertices": nv, "faces": nf, "workspace_MB": round(ws.numel() / 2 ** 20, 1), "build_ms": statistics.median(tb),
            "build_ms_all": tb, "ao_samples": S, "ao_ms": ms_ao, "ao_ms_all": ta, "ao_Mrays_per_s": nv * S / ms_ao / 1e3,
            "inner_vis0": float((vis == 0).float().mean())}


def synced(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def sequence(rounds, nframes=13, target=17000):
    from permuto_sdf_b200.mesh import Mesh, load_mesh_sequence, sequence_files
    N = grid_for(target)
    U, Fc = spheres(N)
    U, Fc = U.double().cpu().numpy(), Fc.cpu().numpy()
    with tempfile.TemporaryDirectory() as d:
        for i in range(nframes):
            V = (U * (1 + 0.02 * i) + np.array([0.01, -0.02, 0.015]) * i).astype(np.float32)
            with open(os.path.join(d, "f_%d.obj" % i), "w") as f:
                f.writelines("v %.9g %.9g %.9g\n" % tuple(v) for v in V)
                f.writelines("f %d %d %d\n" % tuple(t + 1) for t in Fc)
        load_mesh_sequence(d)
        whole = [synced(lambda: load_mesh_sequence(d))[0] for _ in range(rounds)]
        pts = load_mesh_sequence(d)[0]
        steps = {k: 0.0 for k in ("load", "normalize", "normals_upsample", "ao", "remove", "interpolate_normals", "concat")}
        frames = []
        for i, name in enumerate(sequence_files(os.listdir(d))):
            t, m = synced(lambda: Mesh.load(os.path.join(d, name)))
            steps["load"] += t
            if i == 0:
                t, (s, c) = synced(lambda: (m.normalize_size(), m.normalize_position()))
            else:
                t, _ = synced(lambda: m.scale_mesh(s).translate(-c))
            steps["normalize"] += t
            steps["normals_upsample"] += synced(lambda: m.recalculate_normals().upsample(2, True))[0]
            if i == 0:
                t, mask = synced(lambda: m.ambient_occlusion(100) < 0.01)
                steps["ao"] += t
            steps["remove"] += synced(lambda: m.remove_marked_vertices(mask, False).remove_unreferenced_verts())[0]
            frames.append(m)
        t, meshes = synced(lambda: [a.interpolate(b, j / 20).recalculate_normals() for a, b in zip(frames[:-1], frames[1:]) for j in range(20)])
        steps["interpolate_normals"] = t
        K = len(meshes)
        steps["concat"] = synced(lambda: (torch.cat([torch.cat([m.V, torch.full((m.V.shape[0], 1), k / (K - 1), device="cuda")], 1)
                                                     for k, m in enumerate(meshes)]), torch.cat([m.NV for m in meshes])))[0]
    return {"frames": nframes, "faces_per_frame": int(Fc.shape[0]), "faces_after_loop": int(Fc.shape[0]) * 16,
            "rows": int(pts.shape[0]), "ms": statistics.median(whole), "ms_all": whole, "steps_ms": steps}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--faces", type=int, nargs="*", default=[300000, 1000000, 4000000])
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    gpu = card()
    for target in args.faces:
        print(json.dumps({"bench": "bvh_ao", "gpu": gpu, **bvh_ao(target, args.rounds)}), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "load_mesh_sequence", "gpu": gpu, **sequence(max(1, args.rounds // 2))}), flush=True)


if __name__ == "__main__":
    main()
