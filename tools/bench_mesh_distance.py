"""Time of closest-point queries, the pseudonormal build, signed distances and mesh_distance.

Workload:
  closest   rotated sphere-in-sphere meshes of about --faces faces (bench_mesh_ao.spheres): psdf_mesh_closest_points on a prebuilt BVH for
            --points query counts of two kinds, "near" (surface samples moved by N(0, 0.01) per coordinate, the queries of mesh_distance
            and of a fit's near-surface checks) and "uniform" (uniform in the mesh's bounding box grown by 10 %); then, on the near set, the
            pseudonormal build and psdf_mesh_signed_distance, whose difference from the query is the cost of the sign epilogue. Each time
            is the median over --rounds of CUDA events around the call after one warm-up.
  distance  mesh_distance (1 M samples each way) of the mesh extracted at N = 1024 from the fitted sphere of bench_mesh.py against its
            own Loop-subdivided copy, wall clock ending in a device synchronise, median over --rounds after a warm-up.
  brute     for context, a chunked brute-force closest point in torch (the interior projection or the nearest of the three edges, every
            point against every face, fp32,
            on the GPU) on 4096 near points of the smallest mesh, against the BVH query on the same points.
Prints one JSON line per record with the card name and power limit read in the same run.

    python tools/bench_mesh_distance.py [--faces 300000 1000000 4000000] [--points 1000000 16000000] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tools")]

from bench_mesh import card, fitted_model  # noqa: E402
from bench_mesh_ao import grid_for, spheres  # noqa: E402
from bench_mesh_decimate import events_ms  # noqa: E402


def unwritten(dist2, face):
    """outputs still holding the sentinels written before the call (NaN dist2, face -2): a query that left them is an error"""
    n = int((torch.isnan(dist2) | (face == -2)).sum())
    if n:
        raise RuntimeError("psdf_mesh_closest_points left %d of %d outputs unwritten" % (n, dist2.shape[0]))


def checked_closest(m, p):
    """Mesh.closest_points' query on sentinel-filled outputs -> dist [P]"""
    V, Fc, ws = m._bvh("bench")
    from permuto_sdf_b200._lib import call
    d2 = torch.full((p.shape[0],), float("nan"), device="cuda")
    face = torch.full((p.shape[0],), -2, dtype=torch.int32, device="cuda")
    bary = torch.empty(p.shape[0], 3, device="cuda")
    call("psdf_mesh_closest_points", V.shape[0], Fc.shape[0], p.shape[0], p, V, Fc, ws, d2, face, bary)
    unwritten(d2, face)
    return d2.sqrt()


def query_sets(m, n, gen):
    pts, _ = m._sample_surface("bench", n, 1)
    near = pts + 0.01 * torch.randn(pts.shape, device="cuda", generator=gen)
    lo, hi = m.V.min(0).values, m.V.max(0).values
    lo, hi = lo - 0.1 * (hi - lo), hi + 0.1 * (hi - lo)
    uni = lo + (hi - lo) * torch.rand(n, 3, device="cuda", generator=gen)
    return {"near": near.contiguous(), "uniform": uni.contiguous()}


def closest(target, counts, rounds):
    from permuto_sdf_b200._lib import call, load_library
    from permuto_sdf_b200.mesh import Mesh
    V, Fc = spheres(grid_for(target))
    m = Mesh(V, Fc)
    nv, nf = V.shape[0], Fc.shape[0]
    _, _, ws = m._bvh("bench")
    gen = torch.Generator(device="cuda").manual_seed(0)
    out = []
    for P in counts:
        for kind, p in query_sets(m, P, gen).items():
            d2 = torch.full((P,), float("nan"), device="cuda")
            face = torch.full((P,), -2, dtype=torch.int32, device="cuda")
            bary = torch.empty(P, 3, device="cuda")
            q = lambda: call("psdf_mesh_closest_points", nv, nf, P, p, V, Fc, ws, d2, face, bary)
            q()
            unwritten(d2, face)
            t = [events_ms(q)[0] for _ in range(rounds)]
            ms = statistics.median(t)
            rec = {"faces": nf, "points": P, "kind": kind, "ms": ms, "ms_all": t, "Mqueries_per_s": P / ms / 1e3}
            if kind == "near":
                fn, vn, en = m._pseudonormals("bench")
                pws = torch.empty(int(load_library().psdf_mesh_pseudonormals_workspace_bytes(nv, nf)), dtype=torch.uint8, device="cuda")
                pn = lambda: call("psdf_mesh_pseudonormals", nv, nf, V, Fc, pws, fn, vn, en)
                sdf = torch.empty(P, device="cuda")
                sd = lambda: call("psdf_mesh_signed_distance", nv, nf, P, p, V, Fc, ws, fn, vn, en, d2, face, bary, sdf)
                pn()
                sd()
                tp = [events_ms(pn)[0] for _ in range(rounds)]
                ts = [events_ms(sd)[0] for _ in range(rounds)]
                rec.update({"pseudonormals_ms": statistics.median(tp), "signed_distance_ms": statistics.median(ts),
                            "sign_epilogue_ms": statistics.median(ts) - ms})
            out.append(rec)
            del p, d2, face, bary
            torch.cuda.empty_cache()
    return out


# a closest point in torch, every point against every face (fp32, the interior projection or the nearest edge; for context only)
def brute_force(p, a, b, c, chunk):
    dot = lambda x, y: (x * y).sum(-1)
    best = torch.empty(p.shape[0], device="cuda")
    ab, ac, bc = b - a, c - a, c - b
    for s in range(0, p.shape[0], chunk):
        x = p[s:s + chunk, None]
        ap, bp, cp = x - a, x - b, x - c
        d1, d2, d3, d4, d5, d6 = dot(ab, ap), dot(ac, ap), dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
        va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
        den = (va + vb + vc).clamp_min(1e-30)
        q = a + ab * (vb / den)[..., None] + ac * (vc / den)[..., None]                    # interior
        e = lambda o, d, t: o + d * t.clamp(0, 1)[..., None]
        edges = [e(a, ab, d1 / (d1 - d3).clamp_min(1e-30)), e(a, ac, d2 / (d2 - d6).clamp_min(1e-30)),
                 e(b, bc, (d4 - d3) / ((d4 - d3) + (d5 - d6)).clamp_min(1e-30))]
        inside = (va >= 0) & (vb >= 0) & (vc >= 0)
        dist = torch.stack([dot(x - y, x - y) for y in edges], 0).amin(0)
        dist = torch.where(inside, dot(x - q, x - q), dist)
        best[s:s + chunk] = dist.amin(1)
    return best


def brute(target, rounds, P=4096, chunk=64):
    from permuto_sdf_b200.mesh import Mesh
    V, Fc = spheres(grid_for(target))
    m = Mesh(V, Fc)
    p = query_sets(m, P, torch.Generator(device="cuda").manual_seed(0))["near"]
    a, b, c = (V[Fc[:, k].long()] for k in range(3))
    run = lambda: brute_force(p, a, b, c, chunk)
    ref = run()
    t = [events_ms(run)[0] for _ in range(max(1, rounds // 2))]
    dist = checked_closest(m, p)
    assert torch.equal(dist, m.closest_points(p)[0])
    tb = [events_ms(lambda: m.closest_points(p))[0] for _ in range(rounds)]
    return {"faces": Fc.shape[0], "points": P, "brute_ms": statistics.median(t), "bvh_ms_with_build": statistics.median(tb),
            "brute_Mqueries_per_s": P / statistics.median(t) / 1e3, "max_abs_diff": float((ref.sqrt() - dist).abs().max())}


def distance(rounds, N=1024):
    from permuto_sdf_b200.mesh import Mesh, extract_mesh_from_sdf_model, mesh_distance
    m = extract_mesh_from_sdf_model(fitted_model(), N, -0.5, 0.5)
    up = Mesh(m.V.clone(), m.F.clone()).upsample(1, True)
    mesh_distance(m, up)
    t = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = mesh_distance(m, up)
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    sa, _ = m._sample_surface("bench", 1_000_000, 0)
    sb, _ = up._sample_surface("bench", 1_000_000, 0)
    assert torch.equal(checked_closest(up, sa), r["dist_a_to_b"]) and torch.equal(checked_closest(m, sb), r["dist_b_to_a"])
    ts = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m._sample_surface("bench", 1_000_000, 0)
        up._sample_surface("bench", 1_000_000, 0)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"N": N, "faces": m.F.shape[0], "faces_subdivided": up.F.shape[0], "samples": 1_000_000, "ms": statistics.median(t),
            "sample_both_ms": statistics.median(ts), "V_absmax": float(m.V.abs().max()), "V_moved_max": float((up.V[:m.V.shape[0]] - m.V).abs().max()),
            "ms_all": t, **{k: r[k] for k in ("accuracy", "completeness", "chamfer", "hausdorff")}}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--faces", type=int, nargs="*", default=[300000, 1000000, 4000000])
    ap.add_argument("--points", type=int, nargs="*", default=[1000000, 16000000])
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    gpu = card()
    for target in args.faces:
        for rec in closest(target, args.points, args.rounds):
            print(json.dumps({"bench": "closest_points", "gpu": gpu, **rec}), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "brute_force", "gpu": gpu, **brute(args.faces[0], args.rounds)}), flush=True)
    print(json.dumps({"bench": "mesh_distance", "gpu": gpu, **distance(args.rounds)}), flush=True)


if __name__ == "__main__":
    main()
