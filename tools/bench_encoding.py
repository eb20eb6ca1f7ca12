"""Time the standalone permutohedral encoding kernels at every (D, F) the library is built for.

    python tools/bench_encoding.py                             # this tree's library, all 20 pairs
    python tools/bench_encoding.py --roots . ../other --pairs 3,2 4,2    # two builds, alternated round by round
    python tools/bench_encoding.py --deterministic             # also the fixed-point backward and double backward

Problem: N = 2^20 positions uniform in [-0.5, 0.5]^D, L = 16 levels, T = 2^18 rows per level, no concat columns (C = L F), all-ones
window. Per (D, F) and build it times the forward, the backward to the lattice and the positions (one launch, both outputs) and the
double backward (both outputs) with CUDA events around `--launches` back-to-back calls, in `--rounds` rounds; the builds, pairs and
directions alternate inside every round and the median round is reported. It prints ms per call, ns per sample and the algorithmic
bytes per second from shapes, per sample:
    forward          L (D+1) F 4 B gathered + C 4 B written
    backward         C 4 B read + L (D+1) F 4 B gathered + L (D+1) F 4 B reduced into the table + D 4 B written
    double backward  (D + C) 4 B read + L (D+1) F 4 B gathered + L (D+1) F 4 B reduced + C 4 B written
and the card's name and power limit, read in the same run. A pair a build refuses is reported as such.

--deterministic adds the fixed-point twins of the two backward directions (psdf_enc_backward_fx, psdf_enc_double_backward_fx: the
scatter into 64-bit accumulators and the flush that adds them to the float table and clears them), timed in the same rounds as the
float ones, alternating with them. Their bytes per second use the float twin's algorithmic bytes, so the two are directly comparable."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, L, T = 2 ** 20, 16, 2 ** 18
ALL_PAIRS = [(D, F) for D in range(2, 7) for F in (1, 2, 4, 8)]
DIRS = ("forward", "backward", "double_backward")
FX_DIRS = ("forward", "backward", "backward_fx", "double_backward", "double_backward_fx")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown (nvidia-smi unavailable)"


def load(root):
    """the built library of tree `root`, with the argument types of this tree's header (the encoding signatures are unchanged)"""
    sys.path.insert(0, ROOT)
    from permuto_sdf_b200._lib import PROTOS
    lib = ctypes.CDLL(os.path.join(os.path.abspath(root), "permuto_sdf_b200", "libpsdf_b200.so"))
    for name in ("psdf_enc_forward", "psdf_enc_backward", "psdf_enc_double_backward", "psdf_enc_backward_fx",
                 "psdf_enc_double_backward_fx"):
        if not hasattr(lib, name):          # a build from before the deterministic entry points
            continue
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.c_float if k == "float" else ctypes.c_int if k == "int" else ctypes.c_void_p for _, k in PROTOS[name][1]]
    return lib


def bytes_per_sample(D, F):
    C, g = L * F, L * (D + 1) * F * 4
    b = {"forward": g + C * 4, "backward": C * 4 + 2 * g + D * 4, "double_backward": (D + C) * 4 + 2 * g + C * 4}
    b["backward_fx"], b["double_backward_fx"] = b["backward"], b["double_backward"]
    return b


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--roots", nargs="+", default=[ROOT], help="trees whose built libraries run, alternated")
    ap.add_argument("--pairs", nargs="+", default=None, help="D,F pairs (default: all 20)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    ap.add_argument("--deterministic", action="store_true", help="also time the fixed-point backward and double backward")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoding: needs a CUDA device")
    pairs = [tuple(int(v) for v in p.split(",")) for p in a.pairs] if a.pairs else ALL_PAIRS
    libs = [load(r) for r in a.roots]
    dirs = FX_DIRS if a.deterministic else DIRS
    if a.deterministic and not all(hasattr(lib, "psdf_enc_backward_fx") for lib in libs):
        raise SystemExit("bench_encoding: --deterministic needs builds with psdf_enc_backward_fx")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(0)
    times = {}      # (root, D, F, dir) -> [ms per call per round]
    refused = set()
    for D, F in pairs:
        C = L * F
        pos = torch.rand(N, D, device="cuda", generator=g) - 0.5
        lat = (torch.rand(L, T, F, device="cuda", generator=g) - 0.5) * 1e-2
        scale = torch.stack([torch.full((D,), 0.5 * 1.5 ** l) for l in range(L)]).cuda() * 10.0
        shift = torch.randn(L, D, device="cuda", generator=g)
        win = torch.ones(L, device="cuda")
        out = torch.empty(N, C, device="cuda")
        g_out = torch.randn(N, C, device="cuda", generator=g) * 1e-3
        gg = torch.randn(N, D, device="cuda", generator=g) * 1e-3
        g_l, g_p, g_go = torch.zeros_like(lat), torch.empty_like(pos), torch.empty_like(out)
        fx = torch.zeros(L, T, F, dtype=torch.int64, device="cuda") if a.deterministic else None
        head = (N, D, L, F, T, P(pos), P(lat), P(scale), P(shift), P(win), 0, ctypes.c_float(1.0))
        calls = {"forward": lambda lib: lib.psdf_enc_forward(*head, P(out), stream),
                 "backward": lambda lib: lib.psdf_enc_backward(*head, P(g_out), P(g_l), P(g_p), stream),
                 "double_backward": lambda lib: lib.psdf_enc_double_backward(*head, P(gg), P(g_out), P(g_l), P(g_go), stream),
                 "backward_fx": lambda lib: lib.psdf_enc_backward_fx(*head, P(g_out), P(g_l), P(g_p), P(fx), stream),
                 "double_backward_fx": lambda lib: lib.psdf_enc_double_backward_fx(*head, P(gg), P(g_out), P(g_l), P(g_go), P(fx),
                                                                                   stream)}
        for ri, lib in enumerate(libs):
            for d in dirs:                    # warm-up, and the build's refusal of this pair
                if any(calls[d](lib) != 0 for _ in range(3)):
                    refused.add((ri, D, F))
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for ri, lib in enumerate(libs):
                if (ri, D, F) in refused:
                    continue
                for d in dirs:
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    for _ in range(a.launches):
                        calls[d](lib)
                    e.record()
                    torch.cuda.synchronize()
                    times.setdefault((ri, D, F, d), []).append(s.elapsed_time(e) / a.launches)
        del pos, lat, out, g_out, gg, g_l, g_p, g_go, fx
        torch.cuda.empty_cache()
    name = card()
    print("card: %s | N = 2^20, L = 16, T = 2^18, no concat; median of %d rounds x %d launches (min-max of the rounds)" %
          (name, a.rounds, a.launches))
    rows = []
    for D, F in pairs:
        bps = bytes_per_sample(D, F)
        for ri, root in enumerate(a.roots):
            tag = os.path.relpath(os.path.abspath(root), ROOT) if len(a.roots) > 1 else ""
            if (ri, D, F) in refused:
                print("D=%d F=%d %-12s refused by this build" % (D, F, tag))
                continue
            line = "D=%d F=%d %-12s" % (D, F, tag)
            for d in dirs:
                ts = times[(ri, D, F, d)]
                ms = float(np.median(ts))
                rows.append(dict(root=root, D=D, F=F, dir=d, ms=ms, ms_min=min(ts), ms_max=max(ts), ns_per_sample=ms * 1e6 / N,
                                 GBs=bps[d] * N / (ms * 1e-3) / 1e9))
                line += " | %s %.3f ms (%.3f-%.3f) %.2f ns/sample %.0f GB/s" % (d, ms, min(ts), max(ts), ms * 1e6 / N,
                                                                               bps[d] * N / (ms * 1e-3) / 1e9)
            print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump({"card": name, "N": N, "L": L, "T": T, "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
