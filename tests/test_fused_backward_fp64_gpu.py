"""The three fused training backwards (csrc/fused_sdf_bwd.cu, fused_rgb_bwd.cu, fused_bg.cu) against the fp64 reference of the same
operations (oracle/backward_fp64.py), block by block: the lattice gradient per level, W and b per layer, the per-sample outputs of the
colour backward. Every case runs with float atomics and in deterministic mode (64-bit fixed point on the 2^-34 grid), from zeroed and
from pre-filled gradient buffers (the += contract). The C ABI is driven directly, so sets, NULL upstreams and pre-filled buffers are
under the test's control.

Bounds, per gradient tensor block:
  * max|got - ref| / max|ref| <= 1e-3;
  * per element |got_i - ref_i| <= 1e-3 A_i + 1e-4 A'_i + 1e-5 max_block(A) (+ the deterministic rounding budget), A_i = sum over the
    contributions of |contribution| (lattice: per table entry; W: |zbar|^T |a| (+ the tangent stream's); b: sum |zbar|; per-sample
    outputs: |zbar_1| |W_0| through |d normalize|). The A' term (lattice only) and the 1e-5 floor (in place of 1e-6) have one
    reason: the kernels form every product as bf16 hi/lo split GEMMs, whose rounding error is ~2^-17 of the sum of the absolute
    terms, not of the result. Where those terms cancel (an abar_0 or zbar much smaller than |W|^T |zbar|) the error of an element
    exceeds 1e-3 of its own contributions: without these terms the worst elements reached 1.0 - 2.9 times the bound while every
    block stayed within 1e-3. A'_i is A_i with |abar_0| replaced by |zbar_1| |W_0| (and |tabar_0| by |tzbar_1| |W_0|), at 1e-4 (~13x
    above 2^-17); the floor covers a cancelled zbar feeding W_l and b_l;
  * deterministic mode adds n_i 2^-35 (round to nearest on the 2^-34 grid): lattice entries n_i = (sample, vertex) contributions,
    colour / background weights one rounding per tile, SDF weights one per CTA that ran a tile, biases one per 32-row warp and tile;
    elements whose |ref| exceeds the budget must be non-zero;
  * float mode: the non-zero lattice entries are exactly the reference's.
`pytest -s` prints the observed per-block error and the worst per-element ratio err / bound of every case."""
import contextlib
import math

import numpy as np
import pytest
import torch

from oracle import backward_fp64 as R

pytestmark = pytest.mark.gpu
FX = 2.0 ** -35


def _aggregate_below_scale():
    """kAggregateBelowScale of fused_common.cuh: levels whose scale factor is below it aggregate a warp's lanes with match_any"""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "permuto_sdf_b200", "csrc", "fused_common.cuh")).read()
    return float(re.search(r"constexpr float kAggregateBelowScale = ([0-9.]+)f;", src).group(1))


AGG = _aggregate_below_scale()
REPORT = []


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\n%-58s %-6s %-14s %12s %12s" % ("case", "mode", "block", "max rel", "worst ratio"))
        for r in REPORT:
            print("%-58s %-6s %-14s %12.3e %12.3e" % r)


def sms():
    return min(torch.cuda.get_device_properties(0).multi_processor_count, 132)


@contextlib.contextmanager
def mode(m, lattice_entries):
    from permuto_sdf_b200._lib import call
    if m == "det":
        call("psdf_set_deterministic", 1, int(lattice_entries), 64 ** 3)
    try:
        yield
    finally:
        if m == "det":
            call("psdf_set_deterministic", 0, 0, 0)


# ------------------------------------------------------------------------------------------------ inputs
def positions(layout, N, g, D=3):
    """sample layouts: uniform random points; rays of 64 consecutive samples 1/128 of the bounding sphere's diameter apart; every
    sample on one point; uniform points whose last (ragged) warp's valid lanes all sit on one point"""
    if layout == "uniform" or layout == "ragged":
        p = (torch.rand(N, 3, generator=g) - 0.5) * 0.9
        if layout == "ragged":
            tail = N % 32 or 32
            p[N - tail:] = p[N - tail]
    elif layout == "ray":
        nr = (N + 63) // 64
        o = (torch.rand(nr, 3, generator=g) - 0.5) * 0.5
        d = torch.nn.functional.normalize(torch.randn(nr, 3, generator=g), dim=1)
        t = torch.arange(64, dtype=torch.float32) * (1.0 / 128)
        p = (o[:, None, :] + t[None, :, None] * d[:, None, :]).reshape(-1, 3)[:N]
    elif layout == "same":
        p = ((torch.rand(1, 3, generator=g) - 0.5) * 0.9).expand(N, 3)
    if D == 4:      # NeRF++ parametrisation: a unit direction and an inverse distance
        p = torch.cat([torch.nn.functional.normalize(p + 1e-3, dim=1), torch.rand(1 if layout == "same" else N, 1, generator=g).expand(N, 1)], 1)
    return p.contiguous()


def window(L, kind):
    """fully open, or in mid-ramp with one partially weighted level followed by closed ones"""
    if kind == "open":
        return R.window_of(L, 1.0)
    t = (math.floor(0.6 * L) + 0.6) / L
    w = R.window_of(L, t)
    assert ((w > 0) & (w < 1)).any() and (w == 0).any()
    return w


def assert_both_sides_of_aggregation(scale):
    s = scale[:, 0]
    assert bool((s < AGG).any()) and bool((s >= AGG).any()), "levels on both sides of kAggregateBelowScale"


def cu(t):
    return t.detach().float().contiguous().cuda()


# ------------------------------------------------------------------------------------------------ checks
def check(case, m, name, got, ref, A, nround=0.0, init=None, support=False, A_terms=None):
    got = got.detach().double().cpu()
    ref, A = ref.detach().double().cpu(), A.detach().double().cpu()
    slack = 0.0
    if init is not None:
        slack = 2.0 ** -23 * got.abs()          # one fp32 rounding of init + gradient
        got = got - init.detach().double().cpu()
    det = m == "det"
    budget = nround * FX if det else 0.0
    if isinstance(budget, torch.Tensor):
        budget = budget.double().cpu()
    err = (got - ref).abs()
    bound = 1e-3 * A + 1e-5 * float(A.max()) + budget + slack
    if A_terms is not None:
        bound = bound + 1e-4 * A_terms.detach().double().cpu()
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    mref = float(ref.abs().max())
    extra = float(torch.as_tensor(budget).max()) + float(torch.as_tensor(slack).max())
    blk = float(err.max()) / mref if mref > 0 else (0.0 if float(err.max()) <= extra else float("inf"))
    REPORT.append((case, m + ("+=" if init is not None else ""), name, blk, float(ratio.max())))
    assert blk <= 1e-3 + extra / max(mref, 1e-300), (case, m, name, "block", blk)
    worst = int(ratio.reshape(-1).argmax())
    assert float(ratio.max()) <= 1.0, (case, m, name, "element", worst, float(got.reshape(-1)[worst]), float(ref.reshape(-1)[worst]),
                                       float(A.reshape(-1)[worst]))
    if support and not det and init is None:
        assert torch.equal(got != 0, ref != 0), (case, name, "non-zero entries differ from the reference's",
                                                 int(((got != 0) & (ref == 0)).sum()), int(((got == 0) & (ref != 0)).sum()))
    if det and init is None:
        big = ref.abs() > budget
        assert bool((got[big] != 0).all()), (case, name, "deterministic mode rounds a gradient above its budget to zero")


def filled(shape, scale, g):
    return (torch.randn(*shape, generator=g) * scale).float()


# ------------------------------------------------------------------------------------------------ SDF
def sdf_problem(L, hidden, out_dim, T, seed):
    g = torch.Generator().manual_seed(seed)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    dims = [2 * L + 4, hidden, hidden, hidden, out_dim]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    return g, lat, shift, W, b


def sdf_upstream(N, out_dim, g):
    return torch.randn(N, generator=g), torch.randn(N, 3, generator=g), torch.randn(N, out_dim - 1, generator=g)


def run_sdf(sets, L, T, hidden, out_dim, lat, scale, shift, win, W, b, inits):
    """psdf_sdf_fused_backward (one set) or _multi (three) -> (lattice grad, [gW], [gb]) accumulated into copies of `inits`"""
    from permuto_sdf_b200._lib import call, load_library
    lib = load_library()
    blob = torch.empty(int(lib.psdf_sdf_mlp_blob_bytes(2 * L + 4, hidden, out_dim)), dtype=torch.uint8, device="cuda")
    wb = [t for l in range(4) for t in (cu(W[l]), cu(b[l]))]
    call("psdf_sdf_mlp_pack", 2 * L + 4, hidden, out_dim, *wb, blob)
    glat, gW, gb = inits[0].cuda().clone(), [x.cuda().clone() for x in inits[1]], [x.cuda().clone() for x in inits[2]]
    common = (lat.cuda(), scale.cuda(), shift.cuda(), win.cuda(), 1e-3, hidden, out_dim, blob)
    dev = [(s[0], None if s[0] == 0 else cu(s[1]), *[None if u is None else cu(u) for u in s[2:]]) for s in sets]
    if len(sets) == 1:
        n, p, gs, gg, gm = dev[0]
        ws = torch.empty(int(lib.psdf_sdf_fused_backward_workspace_bytes(n)), dtype=torch.uint8, device="cuda")
        call("psdf_sdf_fused_backward", n, L, T, p, *common, gs, gg, gm, glat, ws, *gW, *gb)
    else:
        ws = torch.empty(int(lib.psdf_sdf_fused_backward_multi_workspace_bytes(*[s[0] for s in dev])), dtype=torch.uint8, device="cuda")
        flat = [x for s in dev for x in s]
        call("psdf_sdf_fused_backward_multi", L, T, *common, *flat, glat, ws, *gW, *gb)
    torch.cuda.synchronize()
    return glat.cpu(), [x.cpu() for x in gW], [x.cpu() for x in gb]


def sdf_reference_sets(sets, L, lat, scale, shift, win, W, b):
    """the reference of several sample sets = the sum of the sets' references (A and n add as well)"""
    total = None
    for n, p, gs, gg, gm in sets:
        if n == 0:
            continue
        r = R.sdf_reference(p, lat, scale, shift, win, 1e-3, W, b, gs, gg, gm, device="cuda")
        r["tiles"] = (n + 127) // 128
        if total is None:
            total = r
            continue
        total["lattice"] = [tuple(x + y for x, y in zip(a, c)) for a, c in zip(total["lattice"], r["lattice"])]
        for k in ("W", "b", "A_W", "A_b"):
            total[k] = [x + y for x, y in zip(total[k], r[k])]
        total["tiles"] += r["tiles"]
    return total


def sdf_check_all(case, sets, L, T, hidden, out_dim, lat, scale, shift, win, W, b, g):
    ref = sdf_reference_sets(sets, L, lat, scale, shift, win, W, b)
    tiles = ref["tiles"]
    ctas = min(tiles, sms())
    zeros = (torch.zeros(L, T, 2), [torch.zeros_like(w) for w in W], [torch.zeros_like(x) for x in b])
    for m in ("float", "det"):
        for pre in (False, True):
            if pre:
                init = (torch.stack([filled((T, 2), 0.01 * float(r[0].abs().max()) + 1e-3, g) for r in ref["lattice"]]),
                        [filled(w.shape, 0.01 * float(r.abs().max()) + 1e-3, g) for w, r in zip(W, ref["W"])],
                        [filled(x.shape, 0.01 * float(r.abs().max()) + 1e-3, g) for x, r in zip(b, ref["b"])])
            else:
                init = zeros
            with mode(m, L * T * 2):
                glat, gW, gb = run_sdf(sets, L, T, hidden, out_dim, lat, scale, shift, win, W, b, init)
            ip = init if pre else (None, [None] * 4, [None] * 4)
            for l, (gg, A, n, At) in enumerate(ref["lattice"]):
                check(case, m, "lattice[%d]" % l, glat[l], gg, A, nround=n[:, None].cpu(), init=None if ip[0] is None else ip[0][l],
                      support=True, A_terms=At)
            for l in range(4):
                check(case, m, "W%d" % l, gW[l], ref["W"][l], ref["A_W"][l], nround=ctas, init=ip[1][l])
                check(case, m, "b%d" % l, gb[l], ref["b"][l], ref["A_b"][l], nround=4 * tiles, init=ip[2][l])


SMS_N = ["1", "127", "128sms", "128sms+1", "2*128sms+5"]


def n_of(spec):
    s = sms()
    return {"1": 1, "127": 127, "128sms": 128 * s, "128sms+1": 128 * s + 1, "2*128sms+5": 2 * 128 * s + 5}.get(spec, None) or int(spec)


# (L, hidden, out_dim), T, N, window, layout
SDF_CASES = [
    ((16, 64, 33), 2 ** 18, "2000", "open", "uniform"),
    ((16, 64, 33), 2 ** 18, "1", "mid", "uniform"),
    ((16, 64, 33), 2 ** 10, "127", "open", "ray"),
    ((16, 64, 33), 5003, "128sms", "mid", "uniform"),
    ((16, 64, 33), 2 ** 18, "128sms+1", "open", "ray"),
    ((16, 64, 33), 2 ** 10, "2*128sms+5", "mid", "uniform"),
    ((28, 48, 33), 5003, "3000", "mid", "ray"),
    ((28, 48, 33), 2 ** 18, "128sms+1", "open", "uniform"),
    ((4, 16, 1), 2 ** 10, "1000", "open", "same"),
    ((4, 16, 1), 5003, "127", "mid", "ray"),
    ((8, 32, 33), 2 ** 18, "2000", "mid", "same"),
    ((8, 32, 33), 5003, "389", "open", "ragged"),
    ((16, 64, 33), 2 ** 10, "645", "mid", "ragged"),
]


@pytest.mark.parametrize("shape,T,N,win,layout", SDF_CASES, ids=["L%d-h%d-o%d-T%d-N%s-%s-%s" % (c[0] + c[1:]) for c in SDF_CASES])
def test_sdf_backward_matches_fp64(cuda, shape, T, N, win, layout):
    L, hidden, out_dim = shape
    n = n_of(N)
    g, lat, shift, W, b = sdf_problem(L, hidden, out_dim, T, seed=L * 1000 + n % 997)
    scale = R.level_scales(L, 3)
    assert_both_sides_of_aggregation(scale)
    gs, gg, gm = sdf_upstream(n, out_dim, g)
    sets = [(n, positions(layout, n, g), gs, gg, gm if out_dim > 1 else None)]
    case = "sdf L%d h%d o%d T%d N%d %s %s" % (L, hidden, out_dim, T, n, win, layout)
    sdf_check_all(case, sets, L, T, hidden, out_dim, lat, scale, shift, window(L, win), W, b, g)


@pytest.mark.parametrize("ns", [("129", "0", "64"), ("1", "127", "128sms+1")])
def test_sdf_backward_multi_set_matches_fp64(cuda, ns):
    """three sets in one launch, one of them possibly empty; a NULL g_grad on one set and a NULL g_geom on another"""
    L, hidden, out_dim, T = 16, 64, 33, 5003
    g, lat, shift, W, b = sdf_problem(L, hidden, out_dim, T, seed=77)
    scale = R.level_scales(L, 3)
    sets = []
    for i, spec in enumerate(ns):
        n = n_of(spec)
        gs, gg, gm = sdf_upstream(n, out_dim, g)
        sets.append((n, positions(["uniform", "ray", "uniform"][i], max(n, 1), g)[:n], gs, None if i == 0 else gg, None if i == 2 else gm))
    case = "sdf multi %s" % "/".join(str(s[0]) for s in sets)
    sdf_check_all(case, sets, L, T, hidden, out_dim, lat, scale, shift, window(L, "mid"), W, b, g)


# ------------------------------------------------------------------------------------------------ colour network
def rgb_problem(L, hs, T, seed):
    g = torch.Generator().manual_seed(seed)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    dims = [2 * L + 64] + list(hs) + [3]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    # the matrices the kernel receives: Lipschitz-normalised, with the clamp active on layer 1
    c = [float(w.abs().sum(1).max()) * 2 for w in W]
    c[1] = float(W[1].abs().sum(1).median())
    assert bool((W[1].abs().sum(1) > c[1]).any())
    W = [w * torch.clamp(torch.tensor(ci) / w.abs().sum(1), max=1.0)[:, None] for w, ci in zip(W, c)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    return g, lat, shift, W, b


def run_rgb(acc, N, L, T, hs, pos, dirs, sg, gm, lat, scale, shift, win, W, b, g_out, inits):
    from permuto_sdf_b200._lib import call, load_library
    lib = load_library()
    in_dim = 2 * L + 64
    blob = torch.empty(int(lib.psdf_rgb_mlp_blob_bytes(in_dim, *hs, 3)), dtype=torch.uint8, device="cuda")
    wb = [t for l in range(4) for t in (cu(W[l]), cu(b[l]))]
    call("psdf_rgb_mlp_pack", in_dim, *hs, 3, *wb, blob)
    glat, gsg, ggm = (x.cuda().clone() for x in inits[:3])
    gW, gb = [x.cuda().clone() for x in inits[3]], [x.cuda().clone() for x in inits[4]]
    ws = torch.empty(int(lib.psdf_rgb_fused_backward_workspace_bytes(N)), dtype=torch.uint8, device="cuda")
    call("psdf_rgb_fused_backward_acc" if acc else "psdf_rgb_fused_backward", N, L, T, cu(pos), cu(dirs), cu(sg), cu(gm), 32, lat.cuda(),
         scale.cuda(), shift.cuda(), win.cuda(), 1.0, *hs, blob, cu(g_out), glat, gsg, ggm, ws, *gW, *gb)
    torch.cuda.synchronize()
    return glat.cpu(), gsg.cpu(), ggm.cpu(), [x.cpu() for x in gW], [x.cpu() for x in gb]


# L, (h1, h2, h3), N, layout, window
RGB_CASES = [
    (8, (128, 128, 64), "1", "uniform", "open"),
    (8, (64, 48, 32), "2*128sms+5", "ray", "mid"),
    (16, (128, 128, 64), "127", "same", "mid"),
    (16, (128, 128, 64), "128sms", "ray", "open"),
    (16, (64, 48, 32), "645", "ragged", "open"),
    (24, (128, 128, 64), "128sms+1", "uniform", "mid"),
    (24, (64, 48, 32), "2000", "ray", "open"),
    (28, (128, 128, 64), "2000", "uniform", "mid"),
    (32, (64, 48, 32), "1000", "ray", "open"),
]


@pytest.mark.parametrize("acc", [False, True], ids=["assign", "acc"])
@pytest.mark.parametrize("L,hs,N,layout,win", RGB_CASES, ids=["L%d-h%d.%d.%d-N%s-%s-%s" % ((c[0],) + c[1] + c[2:]) for c in RGB_CASES])
def test_rgb_backward_matches_fp64(cuda, L, hs, N, layout, win, acc):
    T = 5003
    n = n_of(N)
    g, lat, shift, W, b = rgb_problem(L, hs, T, seed=L * 100 + n % 991 + acc)
    scale = R.level_scales(L, 3)
    assert_both_sides_of_aggregation(scale)
    pos = positions(layout, n, g)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    sg, gm, g_out = torch.randn(n, 3, generator=g) * 2, torch.randn(n, 32, generator=g), torch.randn(n, 3, generator=g)
    w = window(L, win)
    ref = R.rgb_reference(pos, dirs, sg, gm, lat, scale, shift, w, 1.0, W, b, g_out, device="cuda")
    tiles = (n + 127) // 128
    case = "rgb L%d h%s N%d %s %s %s" % (L, "/".join(map(str, hs)), n, layout, win, "acc" if acc else "=")
    for m in ("float", "det"):
        for pre in (False, True):
            init = (torch.stack([filled((T, 2), 0.01 * float(r[0].abs().max()) + 1e-3, g) for r in ref["lattice"]]) if pre else torch.zeros(L, T, 2),
                    filled((n, 3), 1.0, g), filled((n, 32), 1.0, g),
                    [filled(x.shape, 0.01 * float(r.abs().max()) + 1e-3, g) if pre else torch.zeros_like(x) for x, r in zip(W, ref["W"])],
                    [filled(x.shape, 0.01 * float(r.abs().max()) + 1e-3, g) if pre else torch.zeros_like(x) for x, r in zip(b, ref["b"])])
            with mode(m, L * T * 2):
                glat, gsg, ggm, gW, gb = run_rgb(acc, n, L, T, hs, pos, dirs, sg, gm, lat, scale, shift, w, W, b, g_out, init)
            for l, (gg, A, cnt, At) in enumerate(ref["lattice"]):
                check(case, m, "lattice[%d]" % l, glat[l], gg, A, nround=cnt[:, None].cpu(), init=init[0][l] if pre else None, support=True,
                      A_terms=At)
            for l in range(4):
                check(case, m, "W%d" % l, gW[l], ref["W"][l], ref["A_W"][l], nround=tiles, init=init[3][l] if pre else None)
                check(case, m, "b%d" % l, gb[l], ref["b"][l], ref["A_b"][l], nround=4 * tiles, init=init[4][l] if pre else None)
            # g_sdf_grad: written (=) or accumulated (_acc) over whatever the buffer held; g_geom is always written
            check(case, m, "g_sdf_grad", gsg, ref["g_sdf_grad"], ref["A_sdf_grad"], init=init[1] if acc else None)
            check(case, m, "g_geom", ggm, ref["g_geom"], ref["A_geom"])


def test_rgb_model_shapes_the_backward_cannot_run_are_refused(cuda):
    """FusedRGB accepts exactly the level counts whose training backward runs (L <= 32, input width 2L + 64 <= 128), and a 32-level
    colour model trains through the fused pair"""
    from permuto_sdf import Sphere
    from permuto_sdf_b200.models import RGB
    with pytest.raises(RuntimeError):
        RGB(3, Sphere(0.5, [0, 0, 0]), 32, 1, nr_levels=36, capacity=2 ** 10).cuda().enable_fused()
    for L in (28, 32):
        m = RGB(3, Sphere(0.5, [0, 0, 0]), 32, 1, nr_levels=L, capacity=2 ** 12).cuda()
        m.fused_head = False
        m.enable_fused()
        pts = (torch.rand(300, 3, device="cuda") - 0.5) * 0.8
        dirs = torch.nn.functional.normalize(torch.randn(300, 3, device="cuda"), dim=1)
        g = torch.randn(300, 3, device="cuda").requires_grad_(True)
        m(pts, dirs, g, torch.randn(300, 32, device="cuda"), 20000).sum().backward()
        assert torch.isfinite(m.encoding.lattice_values.grad).all() and float(m.encoding.lattice_values.grad.abs().max()) > 0


# ------------------------------------------------------------------------------------------------ background network
def run_bg(N, L, T, pos, dirs, lat, scale, shift, win, W, b, g_rgb, g_den, inits):
    from permuto_sdf_b200._lib import call, load_library
    lib = load_library()
    in_dim = 2 * L + 4
    blob = torch.empty(int(lib.psdf_bg_mlp_blob_bytes(in_dim)), dtype=torch.uint8, device="cuda")
    call("psdf_bg_mlp_pack", in_dim, *[t for l in range(7) for t in (cu(W[l]), cu(b[l]))], blob)
    glat, gW, gb = inits[0].cuda().clone(), [x.cuda().clone() for x in inits[1]], [x.cuda().clone() for x in inits[2]]
    ws = torch.empty(int(lib.psdf_bg_fused_backward_workspace_bytes(N)), dtype=torch.uint8, device="cuda")
    call("psdf_bg_fused_backward", N, L, T, cu(pos), cu(dirs), lat.cuda(), scale.cuda(), shift.cuda(), win.cuda(), 1.0, blob, cu(g_rgb),
         cu(g_den), glat, ws, *gW, *gb)
    torch.cuda.synchronize()
    return glat.cpu(), [x.cpu() for x in gW], [x.cpu() for x in gb]


BG_CASES = [(4, "1", 5003, "uniform"), (16, "128sms+1", 2 ** 16, "uniform"), (16, "2000", 5003, "same"), (28, "128sms+1", 5003, "uniform"),
            (28, "1", 2 ** 16, "uniform")]


@pytest.mark.parametrize("L,N,T,layout", BG_CASES, ids=["L%d-N%s-T%d-%s" % c for c in BG_CASES])
def test_background_backward_matches_fp64(cuda, L, N, T, layout):
    """includes trunk layer 3, whose rows the kernel keeps rotated by one (density row last) and un-rotates in its flush"""
    n = n_of(N)
    g = torch.Generator().manual_seed(L * 10 + n % 97)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 4, generator=g) * 10
    dims = [(2 * L + 4, 64), (64, 64), (64, 64), (64, 65), (80, 64), (64, 64), (64, 3)]
    W = [torch.randn(o, i, generator=g) / i ** 0.5 for i, o in dims]
    b = [torch.randn(o, generator=g) * 0.1 for _, o in dims]
    scale = R.level_scales(L, 4)
    pos = positions(layout, n, g, D=4)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    g_rgb, g_den = torch.randn(n, 3, generator=g), torch.randn(n, 1, generator=g)
    w = window(L, "mid")
    ref = R.bg_reference(pos, dirs, lat, scale, shift, w, 1.0, W, b, g_rgb, g_den, device="cuda")
    tiles = (n + 127) // 128
    case = "bg L%d T%d N%d %s" % (L, T, n, layout)
    for m in ("float", "det"):
        for pre in (False, True):
            init = (torch.stack([filled((T, 2), 0.01 * float(r[0].abs().max()) + 1e-3, g) for r in ref["lattice"]]) if pre else torch.zeros(L, T, 2),
                    [filled(x.shape, 0.01 * float(r.abs().max()) + 1e-3, g) if pre else torch.zeros_like(x) for x, r in zip(W, ref["W"])],
                    [filled(x.shape, 0.01 * float(r.abs().max()) + 1e-3, g) if pre else torch.zeros_like(x) for x, r in zip(b, ref["b"])])
            with mode(m, L * T * 2):
                glat, gW, gb = run_bg(n, L, T, pos, dirs, lat, scale, shift, w, W, b, g_rgb, g_den, init)
            for l, (gg, A, cnt, At) in enumerate(ref["lattice"]):
                check(case, m, "lattice[%d]" % l, glat[l], gg, A, nround=cnt[:, None].cpu(), init=init[0][l] if pre else None, support=True,
                      A_terms=At)
            for l in range(7):
                check(case, m, "W%d" % l, gW[l], ref["W"][l], ref["A_W"][l], nround=tiles, init=init[1][l] if pre else None)
                check(case, m, "b%d" % l, gb[l], ref["b"][l], ref["A_b"][l], nround=4 * tiles, init=init[2][l] if pre else None)


# ------------------------------------------------------------------------------------------------ training magnitudes
def _capture_bench_iteration(steps=3):
    """the benchmark's C2 configuration (bench.py: 512 rays x 128 samples, 16 levels, 2^18 entries, 3 x 64 SDF MLP, iteration 20000),
    run eagerly through the direct iteration: the arguments of the last step's fused SDF and colour backward calls, with the weights
    they were packed from (colour: the Lipschitz-normalised matrices, formed by the library's own kernel)"""
    import bench
    from permuto_sdf_b200 import iteration
    from permuto_sdf_b200._lib import call
    from permuto_sdf_b200.train import HyperParams, Trainer
    hp = HyperParams()
    hp.max_nr_samples_per_ray = bench.SAMPLES_PER_RAY - 2 * 16
    hp.nr_samples_imp_sampling = 16
    hp.nr_rays = bench.NR_RAYS
    tr = Trainer(hp, nr_levels=16, capacity=2 ** 18, sdf_hidden=64, nr_images=8, occupancy_resolution=256, seed=0, fused_inference=True,
                 fused_training=True, optimizer="fused", deterministic=True)
    assert tr._direct is not None, tr.execution
    tr.set_analytic_scene()
    tr.iter_nr = 20000
    reel = bench.analytic_reel(8, 600, 800, 1000.0, torch.device("cuda"))
    gen = torch.Generator().manual_seed(1000)
    captured = {}
    orig = iteration.call

    def snap(t):
        return t.detach().clone() if isinstance(t, torch.Tensor) else t

    def spy(name, *args):
        if name == "psdf_sdf_fused_backward_multi":
            lin = tr.model_sdf.fused.lin
            captured["sdf"] = ([snap(a) for a in args[:25]], [snap(l.weight) for l in lin], [snap(l.bias) for l in lin])
        elif name == "psdf_rgb_fused_backward_acc":
            layers = list(tr.model_rgb.mlp.layers)
            weff = []
            for l, lay in enumerate(layers):
                w = lay.weight.detach().contiguous()
                out = torch.empty_like(w)
                orig("psdf_lipschitz_normalize", w.shape[0], w.shape[1], w, tr.model_rgb.mlp.lipshitz_bound_per_layer[l].detach().reshape(1), out)
                weff.append(out)
            captured["rgb"] = ([snap(a) for a in args[:18]], weff, [snap(lay.bias) for lay in layers])
        return orig(name, *args)

    iteration.call = spy
    try:
        for i in range(steps):
            captured.clear()
            pix = bench.central_pixels(bench.NR_RAYS, 600, 800, 300, gen).cuda()
            img = torch.randint(0, 8, (bench.NR_RAYS,), generator=gen, dtype=torch.int32).cuda()
            tr.step_from_reel(reel, pix, img, update_occupancy=(i % 8 == 0))
        torch.cuda.synchronize()
    finally:
        iteration.call = orig
        call("psdf_set_deterministic", 0, 0, 0)
    assert "sdf" in captured and "rgb" in captured
    return captured


def _level_report(what, got_f, got_d, ref_levels):
    """per level: the error of each mode relative to the level's largest reference entry, and the fraction of the float-mode non-zero
    entries that deterministic mode rounds to zero"""
    rows = []
    for l, r in enumerate(ref_levels):
        ref = r[0].double().cpu()
        mref = float(ref.abs().max())
        ef = float((got_f[l].double() - ref).abs().max()) / mref if mref > 0 else 0.0
        ed = float((got_d[l].double() - ref).abs().max()) / mref if mref > 0 else 0.0
        nz = got_f[l] != 0
        lost = float((nz & (got_d[l] == 0)).sum()) / max(int(nz.sum()), 1)
        rows.append((l, mref, ef, ed, int(nz.sum()), lost))
    print("\n%s lattice gradient at training magnitudes (bench C2 configuration, one direct-iteration step)" % what)
    print("%5s %12s %12s %12s %10s %14s" % ("level", "max|ref|", "err float", "err det", "non-zero", "det -> zero"))
    for row in rows:
        print("%5d %12.3e %12.3e %12.3e %10d %14.3e" % row)
    return rows


def test_deterministic_grid_at_training_magnitudes(cuda):
    """the cotangents that reach the fused SDF and colour backward in one training step of the benchmark's configuration, replayed
    with float atomics and in deterministic mode against the fp64 reference: every level of both lattice gradients within 1e-3 in
    both modes (the 2^-34 fixed-point grid is fine enough where the mean-reduced eikonal / curvature terms make the contributions small)"""
    cap = _capture_bench_iteration()
    # ---- SDF: three sample sets (main samples, curvature pass, off-surface points)
    args, W, b = cap["sdf"]
    L, T, lat, scale, shift, win, ps, hidden, out_dim, blob = args[:10]
    sets = []
    for s in range(3):
        n, p, gs, gg, gm = args[10 + 5 * s:15 + 5 * s]
        if n:
            sets.append((n, p[:n].cpu(), None if gs is None else gs[:n].cpu(), None if gg is None else gg[:n].cpu(),
                         None if gm is None else gm[:n].cpu()))
    assert abs(float(ps) - 1e-3) < 1e-9
    ref = sdf_reference_sets(sets, L, lat.cpu(), scale.cpu(), shift.cpu(), win.cpu(), [w.cpu() for w in W], [x.cpu() for x in b])
    zeros = (torch.zeros(L, T, 2), [torch.zeros_like(w).cpu() for w in W], [torch.zeros_like(x).cpu() for x in b])
    got = {}
    for m in ("float", "det"):
        with mode(m, L * T * 2):
            got[m] = run_sdf(sets, L, T, hidden, out_dim, lat, scale.cpu(), shift.cpu(), win.cpu(), [w.cpu() for w in W], [x.cpu() for x in b], zeros)
    rows = _level_report("SDF", got["float"][0], got["det"][0], ref["lattice"])
    for l, mref, ef, ed, _, _ in rows:
        assert ef <= 1e-3 and ed <= 1e-3, ("SDF level", l, ef, ed)
    for l in range(4):
        for m in ("float", "det"):
            e = float((got[m][1][l].double() - ref["W"][l].cpu()).abs().max() / ref["W"][l].abs().max())
            assert e <= 1e-3, ("SDF W", l, m, e)
    # ---- colour network
    args, W_eff, b = cap["rgb"]
    n, L, T, pos, dirs, sg, gm, _, lat, scale, shift, win, ps, h1, h2, h3, blob, g_out = args
    hs = (h1, h2, h3)
    ref = R.rgb_reference(pos[:n].cpu(), dirs[:n].cpu(), sg[:n].cpu(), gm[:n].cpu(), lat.cpu(), scale.cpu(), shift.cpu(), win.cpu(), ps,
                          [w.cpu() for w in W_eff], [x.cpu() for x in b], g_out[:n].cpu(), device="cuda")
    got = {}
    for m in ("float", "det"):
        init = (torch.zeros(L, T, 2), torch.zeros(n, 3), torch.zeros(n, 32), [torch.zeros_like(w).cpu() for w in W_eff],
                [torch.zeros_like(x).cpu() for x in b])
        with mode(m, L * T * 2):
            got[m] = run_rgb(True, n, L, T, hs, pos[:n].cpu(), dirs[:n].cpu(), sg[:n].cpu(), gm[:n].cpu(), lat, scale.cpu(), shift.cpu(),
                             win.cpu(), [w.cpu() for w in W_eff], [x.cpu() for x in b], g_out[:n].cpu(), init)
    rows = _level_report("colour", got["float"][0], got["det"][0], ref["lattice"])
    for l, mref, ef, ed, _, _ in rows:
        assert ef <= 1e-3 and ed <= 1e-3, ("colour level", l, ef, ed)
