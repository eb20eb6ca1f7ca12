"""The fused forward kernels against the fp64 reference of the same operations (oracle/backward_fp64.py: *_forward_reference), element
by element, at the shape limits of every variant: the SDF value + tangent kernel (two-group k_sdf_fused_dual), the value-only
kernel (grad NULL, with and without geom), two sample sets in one launch, the sphere tracer, the colour network (operand blob packed from normalised matrices and by psdf_lipschitz_pack4) and the background network. The C ABI is
driven directly, so kernel variants, NULL outputs and sample sets are under the test's control.

Bounds, per output tensor:
  * max|got - ref| / max|ref| <= 1e-3;
  * per element |got_i - ref_i| <= EPS A_i, A the error scale of the reference (the linearised propagation of absolute terms, see
    oracle/backward_fp64.py) and EPS = 2^-12 (derived and checked against an emulation of the kernels' arithmetic in
    tests/test_forward_fp64_reference_cpu.py);
  * every output buffer carries guard rows past N filled with a NaN sentinel: they must be unchanged, and rows [0, N) finite.
`pytest -s` prints the observed per-tensor error and the worst per-element ratio err / (EPS A) of every case."""
import pytest
import torch

from oracle import backward_fp64 as R
from test_fused_backward_fp64_gpu import cu, n_of, positions, sdf_problem, sms, window

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -12
GUARD = 128                      # guard rows past N of every output buffer
SENTINEL = 0x7FC0DEAD            # a quiet NaN with a payload no kernel writes
REPORT = []

# (L, hidden, out_dim) of the SDF cases: the benchmark shape, the surface fit's, and the limits of launch_forward (hidden 16 / 48,
# out_dim 1 / 17 / 49 / 64, L 28 = in_dim 60 with the concat core the last of Kp = 64)
SDF_SHAPES = [(16, 64, 33), (24, 32, 1), (28, 48, 33), (28, 64, 64), (4, 16, 1), (8, 16, 17), (12, 48, 49), (20, 32, 33)]
RGB_LEVELS = [4, 16, 24, 28, 32]
RGB_HIDDEN = [(128, 128, 64), (64, 48, 32), (128, 64, 16), (16, 16, 16)]
BG_LEVELS = [4, 8, 16, 24, 28]
N_SPECS = ["1", "63", "64", "65", "127", "128", "129", "128sms", "128sms+1", "2*128sms+5"]
T_SIZES = [2 ** 18, 5003, 2 ** 10]
LAYOUTS = ["uniform", "ray", "same", "ragged"]


def n_spec(spec):
    return n_of(spec) if "sms" in spec else int(spec)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\n%-52s %-12s %-8s %12s %12s" % ("case", "kernel", "output", "max rel", "worst ratio"))
        for r in REPORT:
            print("%-52s %-12s %-8s %12.3e %12.3e" % r)
        worst = {}
        for _, k, o, _, w in REPORT:
            worst[(k, o)] = max(worst.get((k, o), 0.0), w)
        print("\nworst element ratio per kernel and output")
        for (k, o), w in sorted(worst.items()):
            print("%-12s %-8s %12.3e" % (k, o, w))


# ------------------------------------------------------------------------------------------------ buffers and checks
def guarded(n, cols, dtype=torch.float32):
    """an output buffer of n rows followed by GUARD rows, every element the NaN sentinel (bytes 0xAB for uint8)"""
    if dtype == torch.uint8:
        return torch.full((n + GUARD,) + ((cols,) if cols else ()), 0xAB, dtype=torch.uint8, device="cuda")
    shape = (n + GUARD,) + ((cols,) if cols else ())
    return torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def rows(buf, n, what):
    """rows [0, n) of a guarded buffer, after checking that the guard rows are untouched and the rows finite"""
    b = buf.cpu()
    if b.dtype == torch.uint8:
        assert bool((b[n:] == 0xAB).all()), (what, "written past N")
        return b[:n]
    assert bool((b[n:].view(torch.int32) == SENTINEL).all()), (what, "written past N", int((b[n:].view(torch.int32) != SENTINEL).sum()))
    assert bool(torch.isfinite(b[:n]).all()), (what, "non-finite rows", int((~torch.isfinite(b[:n])).sum()))
    return b[:n]


def check(case, kernel, name, got, ref, A):
    got, ref, A = got.double().cpu().reshape(ref.shape), ref.detach().double().cpu(), A.detach().double().cpu()
    err = (got - ref).abs()
    bound = EPS * A
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    mref = float(ref.abs().max())
    blk = float(err.max()) / mref if mref > 0 else float(err.max())
    REPORT.append((case, kernel, name, blk, float(ratio.max())))
    assert blk <= 1e-3, (case, kernel, name, "block", blk)
    if float(ratio.max()) > 1.0:
        flat = int(ratio.reshape(-1).argmax())
        cols = ref.shape[1] if ref.dim() > 1 else 1
        r, c = flat // cols, flat % cols
        bad = ratio.reshape(ref.shape[0], -1) > 1.0
        raise AssertionError((case, kernel, name, "element: row %d (in tile %d, in sub-tile %d), column %d" % (r, r % 128, r % 64, c),
                              "got", float(got.reshape(-1)[flat]), "ref", float(ref.reshape(-1)[flat]), "A", float(A.reshape(-1)[flat]),
                              "ratio", float(ratio.max()), "rows over", int(bad.any(1).sum()), "columns over",
                              torch.nonzero(bad.any(0)).reshape(-1).tolist()[:16]))


# ------------------------------------------------------------------------------------------------ SDF
def sdf_blob(L, hidden, out_dim, W, b):
    from permuto_sdf_b200._lib import call, load_library
    blob = torch.empty(int(load_library().psdf_sdf_mlp_blob_bytes(2 * L + 4, hidden, out_dim)), dtype=torch.uint8, device="cuda")
    call("psdf_sdf_mlp_pack", 2 * L + 4, hidden, out_dim, *[t for l in range(4) for t in (cu(W[l]), cu(b[l]))], blob)
    return blob


def run_sdf(L, T, net, sets, hidden, out_dim, blob):
    """psdf_sdf_fused_forward (one set) or _multi (two); sets = [(n, pos, want_grad, want_geom)] -> per set (sdf, grad, geom) rows
    [0, n) (None where not asked for), guard rows checked"""
    from permuto_sdf_b200._lib import call
    lat, scale, shift, win = net
    bufs = []
    for n, p, wg, wm in sets:
        bufs.append((guarded(n, 0), guarded(n, 3) if wg else None, guarded(n, out_dim - 1) if wm and out_dim > 1 else None))
    common = (L, T, lat, scale, shift, win, 1e-3, hidden, out_dim, blob)
    if len(sets) == 1:
        call("psdf_sdf_fused_forward", sets[0][0], L, T, cu(sets[0][1]), *common[2:], *bufs[0])
    else:
        flat = [x for (n, p, _, _), bf in zip(sets, bufs) for x in (n, cu(p), *bf)]
        call("psdf_sdf_fused_forward_multi", *common, *flat)
    torch.cuda.synchronize()
    return [tuple(None if x is None else rows(x, n, nm) for x, nm in zip(bf, ("sdf", "grad", "geom"))) for (n, *_), bf in zip(sets, bufs)]


def sdf_cases():
    """every shape over T, layout and window; the benchmark shape at every N, the others at three N each"""
    out = []
    for si, shape in enumerate(SDF_SHAPES):
        count = len(N_SPECS) if si == 0 else 3
        for k in range(count):
            N = N_SPECS[k] if si == 0 else N_SPECS[(3 * si + k) % len(N_SPECS)]
            out.append((shape, T_SIZES[k % 3], N, LAYOUTS[(si + k) % 4], ["open", "mid"][(si + k // 2) % 2]))
    return out


SDF_CASES = sdf_cases()


@pytest.mark.parametrize("shape,T,N,layout,win", SDF_CASES, ids=["L%d-h%d-o%d-T%d-N%s-%s-%s" % (c[0] + c[1:]) for c in SDF_CASES])
def test_sdf_forward_matches_fp64(cuda, shape, T, N, layout, win):
    """value + tangent kernel (two-group) and the value-only kernel with and without geom, against one reference"""
    L, hidden, out_dim = shape
    n = n_spec(N)
    g, lat, shift, W, b = sdf_problem(L, hidden, out_dim, T, seed=L * 1000 + hidden + n % 997)
    scale, w = R.level_scales(L, 3), window(L, win)
    pos = positions(layout, n, g)
    ref = R.sdf_forward_reference(pos, lat, scale, shift, w, 1e-3, W, b, device="cuda")
    net = (lat.cuda(), scale.cuda(), shift.cuda(), w.cuda())
    blob = sdf_blob(L, hidden, out_dim, W, b)
    case = "sdf L%d h%d o%d T%d N%d %s %s" % (L, hidden, out_dim, T, n, layout, win)
    for kernel in ("dual", "value+geom", "value"):
        tangents, with_geom = kernel == "dual", kernel != "value"
        sdf, grad, geom = run_sdf(L, T, net, [(n, pos, tangents, with_geom)], hidden, out_dim, blob)[0]
        check(case, kernel, "sdf", sdf, ref["sdf"], ref["A_sdf"])
        if tangents:
            check(case, kernel, "grad", grad, ref["grad"], ref["A_grad"])
        if with_geom and out_dim > 1:
            check(case, kernel, "geom", geom, ref["geom"], ref["A_geom"])


MULTI_NS = [("65", "1"), ("64*(2sms+1)", "129"), ("0", "127"), ("1", "0")]
# (grad set 0, grad set 1, geom set 0, geom set 1)
MULTI_OUTPUTS = {"grad-both": (True, True, True, False), "grad-set0": (True, False, False, True), "grad-none": (False, False, True, False)}


@pytest.mark.parametrize("outs", list(MULTI_OUTPUTS), ids=list(MULTI_OUTPUTS))
@pytest.mark.parametrize("ns", MULTI_NS, ids=["%s+%s" % x for x in MULTI_NS])
def test_sdf_forward_multi_set_matches_fp64_and_single_sets(cuda, ns, outs):
    """two sample sets in one launch: sets start on 64-sample sub-tile boundaries (two-group kernel) or 128-sample tile boundaries,
    one CTA's two groups may hold different sets, and a set without grad runs through the value + tangent kernel when the other asks
    for it. Each set against the fp64 reference, and bit for bit against a launch of the same kernel on that set alone."""
    L, hidden, out_dim, T = 16, 64, 33, 5003
    g, lat, shift, W, b = sdf_problem(L, hidden, out_dim, T, seed=91)
    scale, w = R.level_scales(L, 3), window(L, "mid")
    net = (lat.cuda(), scale.cuda(), shift.cuda(), w.cuda())
    blob = sdf_blob(L, hidden, out_dim, W, b)
    wg0, wg1, wm0, wm1 = MULTI_OUTPUTS[outs]
    counts = [64 * (2 * sms() + 1) if s == "64*(2sms+1)" else int(s) for s in ns]
    sets = [(counts[0], positions("uniform", max(counts[0], 1), g)[:counts[0]], wg0, wm0),
            (counts[1], positions("ray", max(counts[1], 1), g)[:counts[1]], wg1, wm1)]
    dual = any(s[2] and s[0] for s in sets)
    got = run_sdf(L, T, net, sets, hidden, out_dim, blob)
    case = "sdf multi %d/%d %s" % (counts[0], counts[1], outs)
    for i, ((n, p, wg, wm), (sdf, grad, geom)) in enumerate(zip(sets, got)):
        if n == 0:
            continue
        ref = R.sdf_forward_reference(p, lat, scale, shift, w, 1e-3, W, b, device="cuda")
        kernel = "multi-dual" if dual else "multi-value"
        check(case + " set%d" % i, kernel, "sdf", sdf, ref["sdf"], ref["A_sdf"])
        if wg:
            check(case + " set%d" % i, kernel, "grad", grad, ref["grad"], ref["A_grad"])
        if wm:
            check(case + " set%d" % i, kernel, "geom", geom, ref["geom"], ref["A_geom"])
        single = run_sdf(L, T, net, [(n, p, wg or dual, wm)], hidden, out_dim, blob)[0]
        assert torch.equal(sdf, single[0]), (case, i, "sdf differs from the single-set launch")
        if wg:
            assert torch.equal(grad, single[1]), (case, i, "grad differs from the single-set launch")
        if wm:
            assert torch.equal(geom, single[2]), (case, i, "geom differs from the single-set launch")


@pytest.mark.parametrize("shape,T", [((16, 64, 33), 2 ** 18), ((28, 48, 33), 5003)], ids=["L16-h64-o33", "L28-h48-o33"])
def test_sphere_trace_step_matches_value_forward(cuda, shape, T):
    """one tracer iteration without an occupancy grid over 4 tiles per CTA slot (the ray queue refills the slots): the traced point
    is x + (d sdf) mult of the value-only forward's sdf in separate fp32 roundings, bit for bit; a ray has converged exactly where
    |sdf| < threshold (wherever the fp64 sdf is farther from the threshold than its bound); every ray is evaluated once"""
    from permuto_sdf_b200._lib import call
    L, hidden, out_dim = shape
    n = 4 * 128 * sms() + 7
    g, lat, shift, W, b = sdf_problem(L, hidden, out_dim, T, seed=5 + L)
    scale, w = R.level_scales(L, 3), window(L, "open")
    pos = positions("uniform", n, g)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    net = (lat.cuda(), scale.cuda(), shift.cuda(), w.cuda())
    blob = sdf_blob(L, hidden, out_dim, W, b)
    ref = R.sdf_forward_reference(pos, lat, scale, shift, w, 1e-3, W, b, device="cuda")
    sdf = run_sdf(L, T, net, [(n, pos, False, False)], hidden, out_dim, blob)[0][0]
    check("trace L%d h%d N%d" % (L, hidden, n), "value", "sdf", sdf, ref["sdf"], ref["A_sdf"])
    thresh = float(ref["sdf"].abs().median())
    mult = 0.7
    pos_out, conv = guarded(n, 3), guarded(n, 0, torch.uint8)
    queue = torch.zeros(8, dtype=torch.int32, device="cuda")
    call("psdf_sdf_sphere_trace", n, L, T, cu(pos), cu(dirs), *net, 1e-3, hidden, out_dim, blob, 1, mult, thresh, None, 1, 1.0,
         [0.0, 0.0, 0.0], 1e3, [0.0, 0.0, 0.0], pos_out, conv, queue)
    torch.cuda.synchronize()
    p_out, c_out = rows(pos_out, n, "pos_out"), rows(conv, n, "converged")
    s = sdf.reshape(n, 1)
    want = pos + (dirs * s) * torch.tensor(mult, dtype=torch.float32)
    assert torch.equal(p_out, want), ("pos_out", int((p_out != want).any(1).sum()))
    sref, A = ref["sdf"].cpu(), ref["A_sdf"].cpu()
    decided = (sref.abs() - thresh).abs() > EPS * A
    assert int(decided.sum()) > n // 2
    assert torch.equal(c_out.bool()[decided], (sref.abs() < thresh)[decided])
    assert int(queue[1]) == n, int(queue[1])


# ------------------------------------------------------------------------------------------------ colour network
def rgb_net(L, hs, T, seed):
    """raw weights W, biases b and Lipschitz bounds c with the clamp active on layer 1 only (softplus(c) at the median row sum)"""
    g = torch.Generator().manual_seed(seed)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    dims = [2 * L + 64] + list(hs) + [3]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    c = [torch.tensor([float(w.abs().sum(1).max()) * 2]) for w in W]
    m = float(W[1].abs().sum(1).median())
    c[1] = torch.tensor([m + torch.log(-torch.expm1(torch.tensor(-m))).item()])           # softplus^-1(m)
    W_eff = [R.lipschitz_weights(w, x) for w, x in zip(W, c)]
    assert bool((W_eff[1] != W[1].double()).any()) and all(torch.equal(W_eff[l], W[l].double()) for l in (0, 2, 3))
    return g, lat, shift, W, b, c, W_eff


def sdf_gradient_rows(n, g):
    """sdf gradients with zero rows, rows of norm 1e-13 (below the 1e-12 normalisation eps) and rows of norm 1e3"""
    sg = torch.randn(n, 3, generator=g) * 2
    u = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    i = torch.arange(n)
    sg[i % 7 == 3] = 0.0
    sg[i % 11 == 5] = u[i % 11 == 5] * 1e-13
    sg[i % 13 == 6] = u[i % 13 == 6] * 1e3
    return sg


def rgb_blobs(L, hs, W, b, c, W_eff):
    from permuto_sdf_b200._lib import call, load_library
    dims = (2 * L + 64, *hs, 3)
    nbytes = int(load_library().psdf_rgb_mlp_blob_bytes(*dims))
    a, p = torch.empty(nbytes, dtype=torch.uint8, device="cuda"), torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    call("psdf_rgb_mlp_pack", *dims, *[t for l in range(4) for t in (cu(W_eff[l]), cu(b[l]))], a)
    call("psdf_lipschitz_pack4", *dims, *[t for l in range(4) for t in (cu(W[l]), cu(b[l]), cu(c[l]))], p)
    return {"normalised": a, "pack4": p}


# L, (h1, h2, h3), N, layout, window
RGB_CASES = [
    (16, (128, 128, 64), "2*128sms+5", "uniform", "open"),
    (16, (16, 16, 16), "129", "ray", "mid"),
    (4, (128, 128, 64), "1", "uniform", "mid"),
    (4, (64, 48, 32), "128sms+1", "ragged", "open"),
    (24, (128, 64, 16), "65", "same", "open"),
    (24, (64, 48, 32), "128sms", "uniform", "mid"),
    (28, (128, 128, 64), "127", "ray", "open"),
    (28, (16, 16, 16), "2*128sms+5", "uniform", "mid"),
    (32, (128, 64, 16), "128sms+1", "ray", "mid"),
    (32, (128, 128, 64), "63", "ragged", "open"),
    (8, (64, 48, 32), "64", "uniform", "open"),
    (12, (128, 64, 16), "128", "ray", "mid"),
]


@pytest.mark.parametrize("L,hs,N,layout,win", RGB_CASES, ids=["L%d-h%d.%d.%d-N%s-%s-%s" % ((c[0],) + c[1] + c[2:]) for c in RGB_CASES])
def test_rgb_forward_matches_fp64(cuda, L, hs, N, layout, win):
    """one reference (W_eff normalised in fp64 from the raw W and c) for the blob packed from normalised matrices and the blob of
    psdf_lipschitz_pack4; multi-tile CTAs stream layer 0's weights again for their next tile"""
    from permuto_sdf_b200._lib import call
    T = 5003
    n = n_spec(N)
    g, lat, shift, W, b, c, W_eff = rgb_net(L, hs, T, seed=L * 100 + sum(hs) + n % 991)
    scale, w = R.level_scales(L, 3), window(L, win)
    pos = positions(layout, n, g)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    sg, gm = sdf_gradient_rows(n, g), torch.randn(n, 32, generator=g)
    ref = R.rgb_forward_reference(pos, dirs, sg, gm, lat, scale, shift, w, 1.0, W_eff, b, device="cuda")
    case = "rgb L%d h%s N%d %s %s" % (L, "/".join(map(str, hs)), n, layout, win)
    for name, blob in rgb_blobs(L, hs, W, b, c, W_eff).items():
        out = guarded(n, 3)
        call("psdf_rgb_fused_forward", n, L, T, cu(pos), cu(dirs), cu(sg), cu(gm), 32, lat.cuda(), scale.cuda(), shift.cuda(), w.cuda(),
             1.0, *hs, blob, out)
        torch.cuda.synchronize()
        check(case, "rgb " + name, "out", rows(out, n, "out"), ref["out"], ref["A_out"])


# ------------------------------------------------------------------------------------------------ background network
BG_CASES = [(4, 5003, "1", "uniform"), (4, 2 ** 16, "2*128sms+5", "uniform"), (8, 5003, "129", "same"), (8, 2 ** 16, "63", "uniform"),
            (16, 2 ** 16, "128sms+1", "uniform"), (16, 5003, "65", "uniform"), (24, 5003, "128sms", "uniform"), (24, 2 ** 16, "127", "same"),
            (28, 2 ** 16, "2*128sms+5", "uniform"), (28, 5003, "64", "uniform")]


@pytest.mark.parametrize("L,T,N,layout", BG_CASES, ids=["L%d-T%d-N%s-%s" % c for c in BG_CASES])
def test_background_forward_matches_fp64(cuda, L, T, N, layout):
    """the trunk's output layer is packed rotated by one row (the density row last); the density row and bias are set so that its
    pre-activation spans [-30, 30] over the samples (both branches of softplus)"""
    from permuto_sdf_b200._lib import call, load_library
    n = n_spec(N)
    g = torch.Generator().manual_seed(L * 10 + n % 97 + T % 7)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 4, generator=g) * 10
    dims = [(2 * L + 4, 64), (64, 64), (64, 64), (64, 65), (80, 64), (64, 64), (64, 3)]
    W = [torch.randn(o, i, generator=g) / i ** 0.5 for i, o in dims]
    b = [torch.randn(o, generator=g) * 0.1 for _, o in dims]
    scale, w = R.level_scales(L, 4), window(L, "mid")
    pos = positions(layout, n, g, D=4)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    args = (pos, dirs, lat, scale, shift, w, 1.0)
    b[3][0] = 0.0
    u = R.bg_forward_reference(*args, W, b, device="cuda")["z_density"].cpu()
    span = float(u.max() - u.min())
    k = 60.0 / span if span > 1e-6 else 1.0
    W[3][0] *= k
    b[3][0] = -30.0 - k * float(u.min())
    ref = R.bg_forward_reference(*args, W, b, device="cuda")
    zd = ref["z_density"]
    assert float(zd.min()) < -29.0 and (n < 2 or span <= 1e-6 or float(zd.max()) > 29.0)
    blob = torch.empty(int(load_library().psdf_bg_mlp_blob_bytes(2 * L + 4)), dtype=torch.uint8, device="cuda")
    call("psdf_bg_mlp_pack", 2 * L + 4, *[t for l in range(7) for t in (cu(W[l]), cu(b[l]))], blob)
    rgb, den = guarded(n, 3), guarded(n, 0)
    call("psdf_bg_fused_forward", n, L, T, cu(pos), cu(dirs), lat.cuda(), scale.cuda(), shift.cuda(), w.cuda(), 1.0, blob, rgb, den)
    torch.cuda.synchronize()
    case = "bg L%d T%d N%d %s" % (L, T, n, layout)
    check(case, "bg", "rgb_raw", rows(rgb, n, "rgb_raw"), ref["rgb_raw"], ref["A_rgb"])
    check(case, "bg", "density", rows(den, n, "density"), ref["density"], ref["A_density"])
