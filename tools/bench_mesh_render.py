"""Time of first-hit ray casting and of mesh rendering from reel cameras.

Workload:
  first_hit  rotated sphere-in-sphere meshes of about --faces faces (bench_mesh_ao.spheres): the 1920 x 1080 rays of one camera at
             distance 1.2 looking at the centre (focal 1500, the rays of PermutoSDF.rays_from_reel_indices), psdf_mesh_first_hit on a
             prebuilt BVH, and psdf_mesh_occluded on the same rays (tnear 0) as the any-hit floor; each the median over --rounds of CUDA
             events around the call after one warm-up, as rays per second.
  render     a 24-frame reel of 800 x 800 sphere_cameras views (focal 700) of the same meshes: psdf_mesh_render with every output, in ms
             per frame, with the 8 x 4 warp tiles of the library and with row order (a copy of mesh_raycast.cu built with -DPSDF_RENDER_ROWS
             into a temporary directory, run on the same workspace; its images must equal the library's bit for bit). The two mappings
             alternate round by round.
  brute      for scale, a chunked brute-force first hit in torch (the same fp32 test of every ray against every face, on the GPU) on
             65536 rays of the 1920 x 1080 camera against a sphere-in-sphere of about 20 k faces, against psdf_mesh_first_hit on the
             same rays.
Prints one JSON line per record with the card name and power limit read in the same run.

    python tools/bench_mesh_render.py [--faces 1000000 4000000] [--rounds 5]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tools")]

from bench_mesh import card  # noqa: E402
from bench_mesh_ao import grid_for, spheres  # noqa: E402
from bench_mesh_decimate import events_ms  # noqa: E402


def camera_rays(H=1080, W=1920, focal=1500.0):
    from permuto_sdf_b200.cameras import TensorReel, look_at
    from permuto_sdf_b200.permuto_sdf import PermutoSDF
    K = torch.tensor([[[focal, 0, W / 2], [0, focal, H / 2], [0, 0, 1]]], dtype=torch.float32, device="cuda")
    eye = torch.tensor([[0.4, 0.5, 1.0]], device="cuda")
    tf = look_at(1.2 * eye / eye.norm())
    reel = TensorReel(torch.zeros(1, 3, H, W, device="cuda"), None, K, tf)
    pix = torch.arange(H * W, dtype=torch.int32, device="cuda")
    o, d, _, _, _ = PermutoSDF.rays_from_reel_indices(reel, pix, torch.zeros_like(pix))
    return o, d


def prebuilt(target):
    from permuto_sdf_b200._lib import call, load_library
    V, Fc = spheres(grid_for(target))
    nv, nf = V.shape[0], Fc.shape[0]
    ws = torch.empty(int(load_library().psdf_mesh_bvh_workspace_bytes(nv, nf)), dtype=torch.uint8, device="cuda")
    call("psdf_mesh_bvh_build", nv, nf, V, Fc, ws)
    return V, Fc, ws


def first_hit(V, Fc, ws, o, d, rounds):
    from permuto_sdf_b200._lib import call
    nv, nf, R = V.shape[0], Fc.shape[0], o.shape[0]
    t = torch.empty(R, device="cuda")
    face = torch.empty(R, dtype=torch.int32, device="cuda")
    bary = torch.empty(R, 3, device="cuda")
    hit = torch.empty(R, dtype=torch.uint8, device="cuda")
    fh = lambda: call("psdf_mesh_first_hit", nv, nf, R, o, d, 0.0, float("inf"), ws, t, face, bary)
    oc = lambda: call("psdf_mesh_occluded", nv, nf, R, o, d, 0.0, float("inf"), ws, hit)
    fh()
    oc()
    tf, to = [], []
    for _ in range(rounds):
        tf.append(events_ms(fh)[0])
        to.append(events_ms(oc)[0])
    if not torch.equal(hit.bool(), face >= 0):
        raise RuntimeError("first_hit and occluded disagree on which rays hit")
    mf, mo = statistics.median(tf), statistics.median(to)
    return {"faces": nf, "rays": R, "hit_fraction": float((face >= 0).float().mean()), "first_hit_ms": mf, "first_hit_ms_all": tf,
            "first_hit_Mrays_per_s": R / mf / 1e3, "occluded_ms": mo, "occluded_ms_all": to, "occluded_Mrays_per_s": R / mo / 1e3}


def rows_library(tmp):
    """mesh_raycast.cu built with the row-order pixel mapping, as a library of its own"""
    import __graft_entry__ as G
    obj, so = os.path.join(tmp, "mesh_raycast_rows.o"), os.path.join(tmp, "libmesh_raycast_rows.so")
    subprocess.run(G.unit_cmd("mesh_raycast.cu", obj, ["-fmad=false", "-DPSDF_RENDER_ROWS"]), check=True, stdout=subprocess.PIPE)
    nvcc = G.shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    subprocess.run([nvcc] + G.ARCH + ["-shared", "-o", so, obj, "-cudart", "static"], check=True, stdout=subprocess.PIPE)
    return ctypes.CDLL(so)


def render(V, Fc, ws, rounds, rows_lib, I=24, H=800, W=800, focal=700.0):
    from permuto_sdf_b200._lib import call
    from permuto_sdf_b200.cameras import sphere_cameras
    K, tf = sphere_cameras(I, H, W, focal)
    nv, nf = V.shape[0], Fc.shape[0]
    outs = {}
    for kind in ("tiles", "rows"):
        outs[kind] = [torch.empty(I, 3, H, W, device="cuda"), torch.empty(I, 1, H, W, device="cuda"), torch.empty(I, 1, H, W, device="cuda"),
                      torch.empty(I, 3, H, W, device="cuda"), torch.empty(I, 1, H, W, dtype=torch.int32, device="cuda")]
    p = lambda x: ctypes.c_void_p(x.data_ptr())

    def rows():
        r = rows_lib.psdf_mesh_render(nv, nf, p(V), p(Fc), None, None, I, H, W, p(K), p(tf), ctypes.c_float(0.0),
                                      ctypes.c_float(float("inf")), p(ws), *[p(x) for x in outs["rows"]],
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if r != 0:
            raise RuntimeError("row-order psdf_mesh_render returned %d" % r)

    run = {"tiles": lambda: call("psdf_mesh_render", nv, nf, V, Fc, None, None, I, H, W, K, tf, 0.0, float("inf"), ws, *outs["tiles"]),
           "rows": rows}
    for k in run:
        run[k]()
    ms = {"tiles": [], "rows": []}
    for _ in range(rounds):
        for k in ("tiles", "rows"):
            ms[k].append(events_ms(run[k])[0] / I)
    for a, b in zip(outs["tiles"], outs["rows"]):
        if not torch.equal(a, b):
            raise RuntimeError("the row-order and tiled mappings rendered different images")
    return {"faces": nf, "frames": I, "H": H, "W": W, "hit_fraction": float(outs["tiles"][1].mean()),
            "tiles_ms_per_frame": statistics.median(ms["tiles"]), "tiles_ms_all": ms["tiles"],
            "rows_ms_per_frame": statistics.median(ms["rows"]), "rows_ms_all": ms["rows"]}


def brute(rounds, nrays=65536, target=20000, chunk=64):
    """first hit of every ray against every face in torch fp32, chunk rays at a time"""
    V, Fc, ws = prebuilt(target)
    o, d = camera_rays()
    sel = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(0))[:nrays].cuda()
    o, d = o[sel].contiguous(), d[sel].contiguous()
    p0, p1, p2 = (V[Fc[:, k].long()] for k in range(3))
    e1, e2 = p1 - p0, p2 - p0

    def torch_first_hit():
        best = []
        for a in range(0, nrays, chunk):
            oc, dc = o[a:a + chunk, None], d[a:a + chunk, None]
            pv = torch.linalg.cross(dc.expand(-1, e2.shape[0], -1), e2[None].expand(oc.shape[0], -1, -1))
            det = (e1[None] * pv).sum(-1)
            inv = 1.0 / det
            tv = oc - p0[None]
            u = (tv * pv).sum(-1) * inv
            qv = torch.linalg.cross(tv, e1[None].expand_as(tv))
            v = (dc * qv).sum(-1) * inv
            t = (e2[None] * qv).sum(-1) * inv
            ok = (det != 0) & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (t > 0)
            best.append(torch.where(ok, t, torch.full_like(t, float("inf"))).min(1))
        return best

    torch_first_hit()
    tt = [events_ms(torch_first_hit)[0] for _ in range(max(1, rounds // 2))]
    r = first_hit(V, Fc, ws, o, d, rounds)
    mt = statistics.median(tt)
    return {"faces": Fc.shape[0], "rays": nrays, "torch_ms": mt, "torch_ms_all": tt, "torch_Mrays_per_s": nrays / mt / 1e3,
            "first_hit_ms": r["first_hit_ms"], "first_hit_Mrays_per_s": r["first_hit_Mrays_per_s"]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--faces", type=int, nargs="*", default=[1000000, 4000000])
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    gpu = card()
    o, d = camera_rays()
    with tempfile.TemporaryDirectory() as tmp:
        rows_lib = rows_library(tmp)
        for target in args.faces:
            V, Fc, ws = prebuilt(target)
            print(json.dumps({"bench": "first_hit", "gpu": gpu, **first_hit(V, Fc, ws, o, d, args.rounds)}), flush=True)
            print(json.dumps({"bench": "render", "gpu": gpu, **render(V, Fc, ws, args.rounds, rows_lib)}), flush=True)
            del V, Fc, ws
            torch.cuda.empty_cache()
    print(json.dumps({"bench": "brute", "gpu": gpu, **brute(args.rounds)}), flush=True)


if __name__ == "__main__":
    main()
