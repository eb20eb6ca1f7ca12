"""Time of the winding-number moment build, winding-number queries and signed distances by either sign.

Workload:
  winding   rotated sphere-in-sphere meshes of about --faces faces (bench_mesh_ao.spheres: two shells wound alike, so |w| is 2 in the
            inner ball, 1 between the shells and 0 outside, and both the far field and the near field run): psdf_mesh_winding_build on a
            prebuilt BVH, then psdf_mesh_winding_number at beta = 2 for --points queries and at beta = +inf (every face, some thousand
            times slower) for the first --exact-points of them, of the "near" and "uniform" sets of bench_mesh_distance.query_sets;
            then Mesh.signed_distance on the near set with sign="pseudonormal" and sign="winding" (each a whole call: BVH build, moments
            or pseudonormals, queries). Each time is the median over --rounds of CUDA events around the
            call after one warm-up. The outputs start as NaN, and a call that leaves one unwritten stops the run.
  brute     for context, a chunked brute-force sum in torch on the GPU (every point against every face: fp32 solid angles, fp64 sum) on
            --brute-points near points of a mesh of about 20 k faces, against the exact and the beta = 2 query on the same points.
Prints one JSON line per record with the card name and power limit read in the same run.

    python tools/bench_mesh_winding.py [--faces 1000000 4000000] [--points 1000000] [--rounds 5]
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tools")]

from bench_mesh import card  # noqa: E402
from bench_mesh_ao import grid_for, spheres  # noqa: E402
from bench_mesh_decimate import events_ms  # noqa: E402
from bench_mesh_distance import query_sets  # noqa: E402


def timed(fn, rounds):
    fn()
    t = [events_ms(fn)[0] for _ in range(rounds)]
    return statistics.median(t), t


def winding(target, P, P_exact, rounds):
    from permuto_sdf_b200._lib import call, load_library
    from permuto_sdf_b200.mesh import Mesh
    V, Fc = spheres(grid_for(target))
    m = Mesh(V, Fc)
    nv, nf = V.shape[0], Fc.shape[0]
    _, _, bvh = m._bvh("bench")
    ws = torch.empty(int(load_library().psdf_mesh_winding_workspace_bytes(nv, nf)), dtype=torch.uint8, device="cuda")
    build_ms, build_all = timed(lambda: call("psdf_mesh_winding_build", nv, nf, V, Fc, bvh, ws), rounds)
    w_centre = float(m.winding_number(V.mean(0, keepdim=True), math.inf))     # the shells' common centre: +-2
    out = [{"faces": nf, "build_ms": build_ms, "build_ms_all": build_all, "workspace_MB": ws.numel() / 2 ** 20, "w_at_centre": w_centre}]
    gen = torch.Generator(device="cuda").manual_seed(0)
    for kind, p in query_sets(m, P, gen).items():
        w = torch.full((P,), float("nan"), device="cuda")
        rec = {"faces": nf, "points": P, "kind": kind}
        for beta, n in ((2.0, P), (math.inf, min(P, P_exact))):
            q = lambda: call("psdf_mesh_winding_number", nv, nf, n, p, bvh, ws, beta, w)
            w.fill_(float("nan"))
            q()
            left = int(torch.isnan(w[:n]).sum())
            if left:
                raise RuntimeError("psdf_mesh_winding_number left %d of %d outputs unwritten" % (left, n))
            key = "beta2" if beta == 2.0 else "exact"
            ms, t = timed(q, rounds)
            rec.update({key + "_points": n, key + "_ms": ms, key + "_ms_all": t, key + "_Mqueries_per_s": n / ms / 1e3})
            if beta == 2.0:
                w2 = w.clone()
                rec["abs_w_histogram"] = {str(k): int(((w.abs() - k).abs() < 0.5).sum()) for k in (0, 1, 2)}
        e = (w2[:n] - w[:n]).abs()
        rec.update({"beta2_max_abs_diff_from_exact": float(e.max()), "beta2_mean_abs_diff_from_exact": float(e.mean())})
        if kind == "near":
            pn_ms, _ = timed(lambda: m.signed_distance(p), rounds)
            wn_ms, _ = timed(lambda: m.signed_distance(p, sign="winding"), rounds)
            rec.update({"signed_distance_pseudonormal_ms": pn_ms, "signed_distance_winding_ms": wn_ms})
        out.append(rec)
        del p, w
        torch.cuda.empty_cache()
    return out


def brute_force(p, a, b, c, chunk):
    """w of every point against every face: fp32 solid angles (Van Oosterom and Strackee), summed in fp64"""
    out = torch.empty(p.shape[0], dtype=torch.float64, device="cuda")
    dot = lambda x, y: (x * y).sum(-1)
    for s in range(0, p.shape[0], chunk):
        x = p[s:s + chunk, None]
        u, v, z = a - x, b - x, c - x
        det = dot(u, torch.cross(v, z, dim=-1))
        lu, lv, lz = u.norm(dim=-1), v.norm(dim=-1), z.norm(dim=-1)
        den = lu * lv * lz + dot(u, v) * lz + dot(v, z) * lu + dot(z, u) * lv
        om = torch.where(det != 0, 2 * torch.atan2(det, den), torch.zeros_like(det))
        out[s:s + chunk] = om.double().sum(1) / (4 * math.pi)
    return out


def brute(P, rounds, target=20000, chunk=16):
    from permuto_sdf_b200.mesh import Mesh
    V, Fc = spheres(grid_for(target))
    m = Mesh(V, Fc)
    p = query_sets(m, P, torch.Generator(device="cuda").manual_seed(0))["near"]
    a, b, c = (V[Fc[:, k].long()] for k in range(3))
    ref = brute_force(p, a, b, c, chunk)
    tb, _ = timed(lambda: brute_force(p, a, b, c, chunk), max(1, rounds // 2))
    te, _ = timed(lambda: m.winding_number(p, math.inf), rounds)
    t2, _ = timed(lambda: m.winding_number(p, 2.0), rounds)
    return {"faces": Fc.shape[0], "points": P, "brute_ms": tb, "exact_ms_with_build": te, "beta2_ms_with_build": t2,
            "exact_max_abs_diff": float((m.winding_number(p, math.inf).double() - ref).abs().max()),
            "beta2_max_abs_diff": float((m.winding_number(p, 2.0).double() - ref).abs().max())}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--faces", type=int, nargs="*", default=[1000000, 4000000])
    ap.add_argument("--points", type=int, default=1000000)
    ap.add_argument("--exact-points", type=int, default=65536)
    ap.add_argument("--brute-points", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh_winding: needs a CUDA device")
    gpu = card()
    for target in args.faces:
        for rec in winding(target, args.points, args.exact_points, args.rounds):
            print(json.dumps({"bench": "winding", "gpu": gpu, **rec}), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "brute_force", "gpu": gpu, **brute(args.brute_points, args.rounds)}), flush=True)


if __name__ == "__main__":
    main()
