"""Compare a training backward (or the SDF forward) of two builds on one fixed, seeded problem at the shape of the C2 training step.

    python tools/ab_backward.py run --kernel sdf --root TREE --out a.npz   # run TREE's library (default: this tree), twice, save the gradients
    python tools/ab_backward.py compare a.npz b.npz                        # gradients of two builds

`--kernel sdf` calls psdf_sdf_fused_backward_multi in deterministic mode with the three sample sets of one training iteration (main
samples with sdf, gradient and geometric-feature upstreams, the curvature pass with gradient upstreams only, 1024 off-surface points with
sdf upstreams only): 16 levels, T = 2^18, hidden 64, out_dim 33, 1030 tiles. It saves the lattice, weight and bias gradients.

`--kernel rgb` calls psdf_rgb_fused_backward_acc (the colour backward of the training step) in deterministic mode: 65 536 samples, 16
levels, T = 2^18, hidden 128 / 128 / 64, 512 tiles. It saves the lattice, weight and bias gradients, g_sdf_grad (accumulated onto a
seeded buffer) and g_geom.

`--kernel sdf_fwd` runs the value + tangent SDF forward of the training step on the same network and sample sets: `--dim 3` calls
psdf_sdf_fused_forward_multi with the main samples (sdf, gradient, geometric features) and the off-surface points (sdf), `--dim 4`
psdf_sdf_fused_forward_dim with space-time positions (the main samples with a seeded time column). It saves every output.

`--kernel enc --dim D --feat F` calls the standalone encoding (psdf_enc_forward, psdf_enc_backward with both outputs,
psdf_enc_double_backward with both outputs) on N_MAIN seeded positions with concat columns, 16 levels, T = 2^18 and a mid-ramp window. It
saves every output. The forward, the positions gradient and grad_grad_out have no reductions across threads and must be bit-identical;
the two lattice gradients (names starting with `atomic_`) are summed with float atomics, whose order changes from run to run (this entry
point has no deterministic mode), so `run` also saves their run-to-run spread and `compare` prints it beside the difference of the two
builds and requires that difference to stay below 1e-5 of the largest value (fp32 sums in another order).

`run` checks that two runs give the same bits and times the call with CUDA events. `compare` requires every saved tensor to be
bit-identical and prints the largest difference of every tensor."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L, T = 16, 2 ** 18
HIDDEN, OUT_DIM = 64, 33                  # SDF network
N_MAIN, N_OFF = 65300, 1024               # 511 + 511 + 8 = 1030 tiles of 128 samples
RGB_HIDDEN, N_RGB, GEOM = (128, 128, 64), 65536, 32     # colour network: 512 tiles


def tiles(kernel):
    if kernel == "rgb":
        return (N_RGB + 127) // 128
    return 2 * ((N_MAIN + 127) // 128) + (N_OFF + 127) // 128


def sdf_problem(torch):
    g = torch.Generator().manual_seed(1234)
    dims = [2 * L + 4, HIDDEN, HIDDEN, HIDDEN, OUT_DIM]
    p = dict(
        lat=(torch.rand(L, T, 2, generator=g) * 2 - 1) * 1e-2,
        scale=torch.stack([torch.full((3,), 0.5 * 1.5 ** l) for l in range(L)]) * 10.0,
        shift=torch.randn(L, 3, generator=g) * 10,
        win=torch.ones(L),
        W=[torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)],
        b=[torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)],
        pos=[(torch.rand(n, 3, generator=g) - 0.5) * 0.9 for n in (N_MAIN, N_MAIN, N_OFF)],
        g_sdf=torch.randn(N_MAIN, generator=g) * 1e-3,
        g_grad=torch.randn(N_MAIN, 3, generator=g) * 1e-3,
        g_geom=torch.randn(N_MAIN, OUT_DIM - 1, generator=g) * 1e-3,
        g_grad_s=torch.randn(N_MAIN, 3, generator=g) * 1e-3,
        g_off=torch.randn(N_OFF, generator=g) * 1e-2,
    )
    return p


def rgb_problem(torch):
    g = torch.Generator().manual_seed(4321)
    dims = [2 * L + 64] + list(RGB_HIDDEN) + [3]
    return dict(
        lat=(torch.rand(L, T, 2, generator=g) * 2 - 1) * 1e-2,
        scale=torch.stack([torch.full((3,), 0.5 * 1.5 ** l) for l in range(L)]) * 10.0,
        shift=torch.randn(L, 3, generator=g) * 10,
        win=torch.ones(L),
        W=[torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)],
        b=[torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)],
        pos=(torch.rand(N_RGB, 3, generator=g) - 0.5) * 0.9,
        dirs=torch.nn.functional.normalize(torch.randn(N_RGB, 3, generator=g), dim=1),
        sdf_grad=torch.randn(N_RGB, 3, generator=g),
        geom=torch.randn(N_RGB, GEOM, generator=g),
        g_out=torch.randn(N_RGB, 3, generator=g) * 1e-3,
        g_sdf_grad0=torch.randn(N_RGB, 3, generator=g) * 1e-3,
    )


def sdf_setup(torch, lib, call, c):
    p = sdf_problem(torch)
    blob = torch.empty(int(lib.psdf_sdf_mlp_blob_bytes(2 * L + 4, HIDDEN, OUT_DIM)), dtype=torch.uint8, device="cuda")
    call("psdf_sdf_mlp_pack", 2 * L + 4, HIDDEN, OUT_DIM, *[c(t) for l in range(4) for t in (p["W"][l], p["b"][l])], blob)
    lat, scale, shift, win = c(p["lat"]), c(p["scale"]), c(p["shift"]), c(p["win"])
    pos = [c(x) for x in p["pos"]]
    segs = [N_MAIN, pos[0], c(p["g_sdf"]), c(p["g_grad"]), c(p["g_geom"]),
            N_MAIN, pos[1], None, c(p["g_grad_s"]), None,
            N_OFF, pos[2], c(p["g_off"]), None, None]
    ws = torch.empty(int(lib.psdf_sdf_fused_backward_multi_workspace_bytes(N_MAIN, N_MAIN, N_OFF)), dtype=torch.uint8, device="cuda")
    glat = torch.zeros(L, T, 2, device="cuda")
    gW = [torch.zeros_like(c(w)) for w in p["W"]]
    gb = [torch.zeros_like(c(x)) for x in p["b"]]

    def once():
        glat.zero_()
        for x in gW + gb:
            x.zero_()
        call("psdf_sdf_fused_backward_multi", L, T, lat, scale, shift, win, 1e-3, HIDDEN, OUT_DIM, blob, *segs, glat, ws, *gW, *gb)

    def result():
        return {"lattice": glat.cpu().numpy(), **{"W%d" % l: gW[l].cpu().numpy() for l in range(4)},
                **{"b%d" % l: gb[l].cpu().numpy() for l in range(4)}}
    return once, result


def sdf_fwd_setup(torch, lib, call, c, dim):
    p = sdf_problem(torch)
    blob = torch.empty(int(lib.psdf_sdf_mlp_blob_bytes(2 * L + 4, HIDDEN, OUT_DIM)), dtype=torch.uint8, device="cuda")
    call("psdf_sdf_mlp_pack", 2 * L + 4, HIDDEN, OUT_DIM, *[c(t) for l in range(4) for t in (p["W"][l], p["b"][l])], blob)
    lat, win = c(p["lat"]), c(p["win"])
    sdf, grad, geom = (torch.zeros(N_MAIN, k, device="cuda") for k in (1, 3, OUT_DIM - 1))
    if dim == 3:
        scale, shift, pos, pos_off = c(p["scale"]), c(p["shift"]), c(p["pos"][0]), c(p["pos"][2])
        sdf_off = torch.zeros(N_OFF, 1, device="cuda")
    else:
        g = torch.Generator().manual_seed(99)
        scale = c(torch.cat([p["scale"], torch.rand(L, 1, generator=g) * 20], 1))
        shift = c(torch.cat([p["shift"], torch.randn(L, 1, generator=g)], 1))
        pos = c(torch.cat([p["pos"][0], torch.rand(N_MAIN, 1, generator=g)], 1))

    def once():
        if dim == 3:
            call("psdf_sdf_fused_forward_multi", L, T, lat, scale, shift, win, 1e-3, HIDDEN, OUT_DIM, blob, N_MAIN, pos, sdf, grad, geom,
                 N_OFF, pos_off, sdf_off, None, None)
        else:
            call("psdf_sdf_fused_forward_dim", 4, N_MAIN, L, T, pos, lat, scale, shift, win, 1e-3, HIDDEN, OUT_DIM, blob, sdf, grad, geom)

    def result():
        r = {"sdf": sdf.cpu().numpy(), "grad": grad.cpu().numpy(), "geom": geom.cpu().numpy()}
        if dim == 3:
            r["sdf_off"] = sdf_off.cpu().numpy()
        return r
    return once, result


def rgb_setup(torch, lib, call, c):
    p = rgb_problem(torch)
    in_dim = 2 * L + 64
    blob = torch.empty(int(lib.psdf_rgb_mlp_blob_bytes(in_dim, *RGB_HIDDEN, 3)), dtype=torch.uint8, device="cuda")
    call("psdf_rgb_mlp_pack", in_dim, *RGB_HIDDEN, 3, *[c(t) for l in range(4) for t in (p["W"][l], p["b"][l])], blob)
    lat, scale, shift, win = c(p["lat"]), c(p["scale"]), c(p["shift"]), c(p["win"])
    pos, dirs, sg, gm, g_out, sg0 = (c(p[k]) for k in ("pos", "dirs", "sdf_grad", "geom", "g_out", "g_sdf_grad0"))
    ws = torch.empty(int(lib.psdf_rgb_fused_backward_workspace_bytes(N_RGB)), dtype=torch.uint8, device="cuda")
    glat = torch.zeros(L, T, 2, device="cuda")
    gsg = torch.zeros(N_RGB, 3, device="cuda")
    ggm = torch.zeros(N_RGB, GEOM, device="cuda")
    gW = [torch.zeros_like(c(w)) for w in p["W"]]
    gb = [torch.zeros_like(c(x)) for x in p["b"]]

    def once():
        glat.zero_()
        gsg.copy_(sg0)
        for x in gW + gb:
            x.zero_()
        call("psdf_rgb_fused_backward_acc", N_RGB, L, T, pos, dirs, sg, gm, GEOM, lat, scale, shift, win, 1e-3, *RGB_HIDDEN, blob, g_out,
             glat, gsg, ggm, ws, *gW, *gb)

    def result():
        return {"lattice": glat.cpu().numpy(), **{"W%d" % l: gW[l].cpu().numpy() for l in range(4)},
                **{"b%d" % l: gb[l].cpu().numpy() for l in range(4)}, "g_sdf_grad": gsg.cpu().numpy(), "g_geom": ggm.cpu().numpy()}
    return once, result


def enc_setup(torch, call, dim, feat):
    g = torch.Generator().manual_seed(2024)
    C = (L + (dim + feat - 1) // feat) * feat
    lat = ((torch.rand(L, T, feat, generator=g) * 2 - 1) * 1e-2).cuda()
    scale = (torch.stack([torch.full((dim,), 0.5 * 1.5 ** l) for l in range(L)]) * 10.0).cuda()
    shift = (torch.randn(L, dim, generator=g) * 10).cuda()
    win = (0.5 * (1 + torch.cos(torch.pi * torch.clip(0.6 * L - torch.arange(L), 0, 1) + torch.pi))).cuda()
    pos = ((torch.rand(N_MAIN, dim, generator=g) - 0.5) * 0.9).cuda()
    g_out = (torch.randn(N_MAIN, C, generator=g) * 1e-3).cuda()
    gg = (torch.randn(N_MAIN, dim, generator=g) * 1e-3).cuda()
    out, g_go = (torch.empty(N_MAIN, C, device="cuda") for _ in range(2))
    g_p = torch.empty(N_MAIN, dim, device="cuda")
    g_l, d_l = torch.zeros_like(lat), torch.zeros_like(lat)
    head = (N_MAIN, dim, L, feat, T, pos, lat, scale, shift, win, 1, 1e-3)

    def once():
        g_l.zero_()
        d_l.zero_()
        call("psdf_enc_forward", *head, out)
        call("psdf_enc_backward", *head, g_out, g_l, g_p)
        call("psdf_enc_double_backward", *head, gg, g_out, d_l, g_go)

    def result():
        return {"out": out.cpu().numpy(), "grad_pos": g_p.cpu().numpy(), "grad_grad_out": g_go.cpu().numpy(),
                "atomic_grad_lattice": g_l.cpu().numpy(), "atomic_dbl_grad_lattice": d_l.cpu().numpy()}
    return once, result


def run(args):
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from permuto_sdf_b200._lib import call, load_library
    lib = load_library()
    assert lib.psdf_device_ok() == 1, "needs a CUDA device"
    c = lambda t: t.float().contiguous().cuda()
    if args.kernel == "sdf_fwd":
        once, result = sdf_fwd_setup(torch, lib, call, c, args.dim)
    elif args.kernel == "enc":
        once, result = enc_setup(torch, call, args.dim, args.feat)
    else:
        once, result = (rgb_setup if args.kernel == "rgb" else sdf_setup)(torch, lib, call, c)
    det = args.kernel not in ("sdf_fwd", "enc")  # the forward has no reductions; the encoding has no deterministic mode
    if det:
        call("psdf_set_deterministic", 1, L * T * 2, 64 ** 3)
    try:
        results = []
        for _ in range(2):
            once()
            torch.cuda.synchronize()
            results.append(result())
        same = all(np.array_equal(results[0][k], results[1][k]) for k in results[0] if not k.startswith("atomic_"))
        for k in [k for k in results[0] if k.startswith("atomic_")]:
            results[0]["spread_" + k] = np.array(np.abs(results[0][k].astype(np.float64) - results[1][k]).max())
        for _ in range(5):
            once()
        reps = 50
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        for _ in range(reps):
            once()
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / reps
    finally:
        if det:
            call("psdf_set_deterministic", 0, 0, 0)
    name = torch.cuda.get_device_name(0)
    if args.kernel == "enc":
        what = "forward + backward + double backward, D = %d, F = %d, %d samples" % (args.dim, args.feat, N_MAIN)
    elif args.kernel == "sdf_fwd":
        what = "forward, D = %d" % args.dim
    else:
        what = "zeroing + backward, deterministic, %d tiles" % tiles(args.kernel)
    print("%s [%s]: two runs bit-identical: %s | %.3f ms per call (%s) on %s" % (args.root, args.kernel, same, ms, what, name))
    np.savez(args.out, **results[0])
    return 0 if same else 1


def compare(args):
    a, b = np.load(args.a), np.load(args.b)
    ok = sorted(a.files) == sorted(b.files)
    for k in sorted(set(a.files) & set(b.files)):
        if k.startswith("spread_"):
            continue
        x, y = a[k].astype(np.float64), b[k].astype(np.float64)
        d = float(np.abs(x - y).max())
        same = np.array_equal(a[k], b[k])
        if k.startswith("atomic_"):        # float-atomic sums: the order of the additions changes from run to run
            spread = max(float(a["spread_" + k]), float(b["spread_" + k]))
            good = d <= 1e-5 * float(np.abs(x).max())
            print("%-24s max |diff| %.3e  max |value| %.3e  run-to-run spread %.3e  below 1e-5 relative: %s" % (k, d, float(np.abs(x).max()),
                                                                                                              spread, good))
        else:
            good = same
            print("%-24s max |diff| %.3e  max |value| %.3e  bit-identical: %s" % (k, d, float(np.abs(x).max()), good))
        ok &= good
    print("PASS" if ok else "FAIL")
    return 0 if ok else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("run")
    r.add_argument("--kernel", choices=["sdf", "rgb", "sdf_fwd", "enc"], default="sdf",
                   help="which training backward (or the SDF forward, or the standalone encoding) runs")
    r.add_argument("--dim", type=int, choices=[2, 3, 4, 5, 6], default=3, help="input width (--kernel sdf_fwd: 3 or 4; --kernel enc: 2..6)")
    r.add_argument("--feat", type=int, choices=[1, 2, 4, 8], default=2, help="features per level of the encoding (--kernel enc)")
    r.add_argument("--root", default=ROOT, help="tree whose permuto_sdf_b200 package (and built library) runs")
    r.add_argument("--out", required=True)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    return run(args) if args.cmd == "run" else compare(args)


if __name__ == "__main__":
    sys.exit(main())
