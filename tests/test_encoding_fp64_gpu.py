"""The permutohedral encoding kernels (csrc/encoding.cu) against the fp64 reference of oracle/encoding_fp64.py, element by element,
at every supported (D, F) pair and through every C-ABI entry point: psdf_enc_forward, psdf_enc_backward (lattice only, positions only,
both), psdf_enc_double_backward (lattice only, grad_out only, both) and the fixed-point twins.

Every output tensor is held to
  * max |got - ref| / max |ref| <= 1e-3 (where the reference cancels to ~0, e.g. at T = 1, the largest per-element bound times 1e3
    stands in for max |ref|);
  * |got - ref| <= EPS A per element, EPS and A as derived in oracle/encoding_fp64.py (closed levels and concat pad columns have A = 0,
    so they must be exact zeros);
  * lattice gradients per entry: (n_e + M) u (A_e + |prefill|) in float, sum(2^-35 + M u |c|) + u |total| + u |ref| in fixed point;
    a table entry no sample reaches keeps its prefilled value bit for bit;
  * NaN guard rows before and after every output unchanged, and every row of [0, N) written and finite.
The cases spread N over {1, 31, 32, 33, 4097, 40003}, L over {1, 5, 7, 32}, T over {1, 3, 4099, 2^14, 2^20 + 7}, concat off and on
(with several groups and with pad columns), the window over none / all open / partly open / closed levels, and the positions over a
uniform box, clusters with exact duplicate rows (warp aggregation), a dyadic grid on power-of-two scales (positions on lattice
vertices and faces: rank ties and zero weights), negative positions and large positions ((x + shift) scale up to ~2e5).
`pytest -s` prints, per case and tensor, the tensor-wide ratio and the worst per-element ratio err / bound."""
import collections

import numpy as np
import pytest
import torch

from oracle import encoding_fp64 as X
from oracle import encoding_oracle as eo

pytestmark = pytest.mark.gpu

PAIRS = [(D, F) for D in range(2, 7) for F in (1, 2, 4, 8)]
GUARD = 4
Case = collections.namedtuple("Case", "D F N L T concat window layout")

_NS = [1, 31, 32, 33, 4097, 40003]
_LS = [1, 5, 7, 32]
_TS = [1, 3, 4099, 2 ** 14, 2 ** 20 + 7]
_WINDOWS = ["none", "open", "partial", "closed"]
_LAYOUTS = ["uniform", "clustered", "lattice", "negative", "large"]
CASES = [Case(D, F, _NS[i % 6], _LS[(i // 3) % 4], _TS[(i * 2) % 5], i % 4 != 3, _WINDOWS[i % 4], _LAYOUTS[(i + i // 5) % 5])
         for i, (D, F) in enumerate(PAIRS)]


def positions(c, g):
    D, N = c.D, c.N
    if c.layout == "clustered":
        centres = torch.rand(40, D, generator=g) - 0.5
        cid = torch.randint(0, 40, (N,), generator=g).sort().values
        pos = centres[cid] + 2e-3 * torch.randn(N, D, generator=g)
        if N >= 8:
            pos[N // 2:N // 2 + N // 8] = pos[:N // 8]
        return pos
    if c.layout == "lattice":
        return torch.randint(-12, 13, (N, D), generator=g).float() / 4
    if c.layout == "negative":
        return -(torch.rand(N, D, generator=g) * 2 + 0.5)
    if c.layout == "large":
        return torch.rand(N, D, generator=g) * 5 + 5
    return torch.rand(N, D, generator=g) - 0.5


def level_consts(c, g):
    """scale [L, D], shift [L, D]: powers of two without shift for the lattice layout (exact elevation, exact ties), else the
    geometric sigmas 1 .. 1e-4 and random shifts as PermutoEncoding makes them"""
    if c.layout == "lattice":
        scale = (2.0 ** (torch.arange(c.L) % 4 - 1)).float()[:, None].expand(c.L, c.D).contiguous()
        return scale, torch.zeros(c.L, c.D)
    scale = eo.scale_factor([float(s) for s in np.geomspace(1.0, 1e-4, num=c.L)], c.D)
    shift = torch.randn(c.L, c.D, generator=g) * 10
    if c.layout == "negative":
        shift = -shift.abs()
    return scale, shift


def window_of(c):
    if c.window == "none":
        return None
    if c.window == "open":
        return torch.ones(c.L)
    w = eo.coarse2fine(c.L, 0.55)
    if c.window == "closed":
        w[c.L // 2:] = 0.0
        w[0] = 0.0
    return w


_PLANS = {}


def setup(i):
    """inputs and the fp64 reference of case i (the CPU plan is the slow part: cached per case)"""
    c = CASES[i]
    if i not in _PLANS:
        g = torch.Generator().manual_seed(1000 + i)
        pos = positions(c, g)
        scale, shift = level_consts(c, g)
        lat = torch.rand(c.L, c.T, c.F, generator=g) * 2 - 1
        C = c.L * c.F + X.n_extra(c.D, c.F, c.concat)
        g_out, gg = torch.randn(c.N, C, generator=g), torch.randn(c.N, c.D, generator=g)
        pre, pre2 = torch.randn(c.L, c.T, c.F, generator=g), torch.randn(c.L, c.T, c.F, generator=g)
        plan = X.plan_of(pos, scale, shift, c.T, "cuda")
        _PLANS[i] = (pos, scale, shift, lat, g_out, gg, pre, pre2, plan)
    return c, _PLANS[i]


def guarded(shape, fill=float("nan")):
    rows = shape[0]
    rest = tuple(shape[1:])
    buf = torch.full((rows + 2 * GUARD,) + rest, fill, device="cuda")
    return buf, buf[GUARD:GUARD + rows]


def guards_intact(buf):
    return bool(torch.isnan(buf[:GUARD]).all()) and bool(torch.isnan(buf[buf.shape[0] - GUARD:]).all())


def guarded_table(pre):
    """a prefilled [L, T, F] table with NaN guard rows (of F floats) before and after it"""
    L, T, F = pre.shape
    buf = torch.full((L * T + 2 * GUARD, F), float("nan"), device="cuda")
    view = buf[GUARD:GUARD + L * T].view(L, T, F)
    view.copy_(pre)
    return buf, view


def rel_err(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).abs().max() / (ref.abs().max() + 1e-30)) if ref.numel() else 0.0


def check_dense(tag, buf, got, ref, A, eps):
    """an [N, C] or [N, D] output: guards, finite rows, the tensor-wide ratio and the per-element bound"""
    torch.cuda.synchronize()
    assert buf is None or guards_intact(buf), tag + ": wrote outside its rows"
    assert bool(torch.isfinite(got).all()), tag + ": a row was not written or is not finite"
    # a reference that cancels to ~0 (T = 1: every vertex on one row, so the weights' derivatives sum to zero) is judged per element
    e = float((got.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e3 * float((eps * A).max()), 1e-30) if ref.numel() else 0.0
    w = X.worst((got.double() - ref).abs(), eps * A)
    print("  %-22s rel %.2e  worst err/(EPS A) %.3f" % (tag, e, w))
    assert e <= 1e-3, (tag, e)
    assert w <= 1.0, (tag, w)
    zero = A == 0
    assert bool((got[zero] == 0).all()), tag + ": a closed level or pad column is not an exact zero"


def check_table(tag, buf, got, ref, A, n, pre, m, fx):
    torch.cuda.synchronize()
    assert guards_intact(buf), tag + ": wrote outside the table"
    got64 = got.double()
    bound = X.lattice_bound_fx(ref, A, n, m) if fx else X.lattice_bound(ref, A, n, pre, m)
    # where the contributions cancel (T = 1: every vertex on one row) the largest per-entry bound stands in for max |ref|
    e = float((got64 - ref).abs().max()) / max(float(ref.abs().max()), 1e3 * float(bound.max()), 1e-30)
    w = X.worst((got64 - ref).abs(), bound)
    print("  %-22s rel %.2e  worst err/bound %.3f" % (tag, e, w))
    assert e <= 1e-3, (tag, e)
    assert w <= 1.0, (tag, w)
    untouched = n == 0
    assert torch.equal(got[untouched], pre[untouched]), tag + ": an entry no sample reaches changed"


@pytest.mark.parametrize("i", range(len(CASES)), ids=lambda i: "D%d-F%d" % CASES[i][:2])
def test_every_entry_point_against_fp64(cuda, i):
    from permuto_sdf_b200 import call
    c, (pos, scale, shift, lat, g_out, gg, pre, pre2, plan) = setup(i)
    print("\n%s" % (c,))
    D, F, N, L, T = c.D, c.F, c.N, c.L, c.T
    win = window_of(c)
    ref = X.reference(plan, lat, win, c.concat, 0.5, g_out, gg, pos, prefill=pre.cuda(), prefill2=pre2.cuda())
    C = ref["out"].shape[1]
    dpos, dlat, dgo, dgg = pos.cuda(), lat.cuda(), g_out.cuda(), gg.cuda()
    dpre, dpre2 = pre.cuda(), pre2.cuda()
    args = (N, D, L, F, T, dpos, dlat, scale.cuda(), shift.cuda(), None if win is None else win.cuda(), int(c.concat), 0.5)
    ws = torch.zeros(L, T, F, dtype=torch.int64, device="cuda")

    buf, out = guarded((N, C))
    call("psdf_enc_forward", *args, out)
    check_dense("forward", buf, out, ref["out"], ref["A_out"], X.EPS_FWD)

    for fn, extra, fx in (("psdf_enc_backward", (), False), ("psdf_enc_backward_fx", (ws,), True)):
        for want_l, want_p in ((True, False), (False, True), (True, True)):
            tb, g_l = guarded_table(dpre) if want_l else (None, None)
            pb, g_p = guarded((N, D)) if want_p else (None, None)
            call(fn, *args, dgo, g_l, g_p, *extra)
            tag = "%s[%s%s]" % (fn[9:], "L" if want_l else "", "P" if want_p else "")
            if want_l:
                check_table(tag + " lattice", tb, g_l, ref["lat"], ref["lat_A"], ref["lat_n"], dpre, X.M_LAT, fx)
            if want_p:
                check_dense(tag + " pos", pb, g_p, ref["pos_grad"], ref["A_pos"], X.EPS_POS)
            assert int(ws.count_nonzero()) == 0, "the fixed-point accumulators were not cleared"

    for fn, extra, fx in (("psdf_enc_double_backward", (), False), ("psdf_enc_double_backward_fx", (ws,), True)):
        for want_l, want_g in ((True, False), (False, True), (True, True)):
            tb, g_l = guarded_table(dpre2) if want_l else (None, None)
            ob, g_go = guarded((N, C)) if want_g else (None, None)
            call(fn, *args, dgg, dgo, g_l, g_go, *extra)
            tag = "%s[%s%s]" % (fn[9:], "L" if want_l else "", "G" if want_g else "")
            if want_l:
                check_table(tag + " lattice", tb, g_l, ref["dlat"], ref["dlat_A"], ref["dlat_n"], dpre2, X.M_DLAT, fx)
            if want_g:
                check_dense(tag + " grad_out", ob, g_go, ref["ggo"], ref["A_ggo"], X.EPS_GGO)
            assert int(ws.count_nonzero()) == 0, "the fixed-point accumulators were not cleared"


@pytest.mark.parametrize("T", [1, 3, 4099, 5003, 2 ** 20 + 7])
@pytest.mark.parametrize("D,F", [(2, 8), (3, 1), (4, 2), (5, 4), (6, 1)])
def test_hashed_rows_and_weights_exact(cuda, D, F, T):
    """with g = 1 and an open window the backward's lattice gradient is the sum of the weights that reach each row: the touched rows
    are exactly the oracle's hashed rows (non-power-of-two T: the conditional subtraction of the division-free h mod T), and an entry
    reached once holds the oracle's fp32 weight bit for bit"""
    from permuto_sdf_b200 import call
    L, N = 5, 4097
    g = torch.Generator().manual_seed(D * 100 + F * 10 + T % 97)
    pos = torch.cat([torch.rand(N - 1024, D, generator=g) - 0.5, torch.randint(-12, 13, (1024, D), generator=g).float() / 4])
    scale = eo.scale_factor([float(s) for s in np.geomspace(1.0, 1e-3, num=L)], D)
    shift = torch.randn(L, D, generator=g) * 10
    plan = X.plan_of(pos, scale, shift, T, "cuda")
    C = L * F
    ref = X.reference(plan, torch.zeros(L, T, F), None, False, 1.0, torch.ones(N, C), None, pos)
    g_l = torch.zeros(L, T, F, device="cuda")
    call("psdf_enc_backward", N, D, L, F, T, pos.cuda(), torch.zeros(L, T, F, device="cuda"), scale.cuda(), shift.cuda(), None, 0, 1.0,
         torch.ones(N, C, device="cuda"), g_l, None)
    torch.cuda.synchronize()
    reached = ref["lat_A"][:, :, 0] > 0
    for k in range(F):
        assert torch.equal(g_l[:, :, k] != 0, reached), "column %d: touched rows differ from the oracle's hashed rows" % k
    once = ref["lat_n"] == 1
    assert int(once.sum()) > 0 or T < 5000
    assert torch.equal(g_l.double()[once], ref["lat"][once]), "a weight differs from the oracle's fp32 weight"
    if T > 2 ** 20:
        assert int(once[:, :, 0].sum()) > 1000


def _free_bytes():
    return torch.cuda.mem_get_info()[0]


def test_output_above_2_31_elements(cuda):
    """D = 2, F = 8, L = 32, concat: C = 264 columns, N = 2^23 + 33 rows, 2.2e9 elements per [N, C] tensor (8.9 GB). The forward output,
    the positions gradient (reads grad_out) and grad_grad_out are checked on the first block, the blocks around element 2^31 and the
    last partial block. Needs ~27 GB of free device memory (three [N, C] buffers)."""
    from permuto_sdf_b200 import call
    D, F, L, T, N = 2, 8, 32, 2 ** 14, 2 ** 23 + 33
    C = (L + 1) * F
    need = 3 * (N + 2 * GUARD) * C * 4 + (2 << 30)
    if _free_bytes() < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 2 ** 30, _free_bytes() / 2 ** 30))
    assert N * C > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(5)
    pos = torch.rand(N, D, device="cuda", generator=g) - 0.5
    gg = torch.randn(N, D, device="cuda", generator=g)
    lat = torch.rand(L, T, F, device="cuda", generator=g) * 2 - 1
    scale = eo.scale_factor([float(s) for s in np.geomspace(1.0, 1e-4, num=L)], D)
    shift = torch.randn(L, D, generator=torch.Generator().manual_seed(6)) * 10
    win = eo.coarse2fine(L, 0.7)
    args = (N, D, L, F, T, pos, lat, scale.cuda(), shift.cuda(), win.cuda(), 1, 0.5)
    r0 = 2 ** 31 // C
    rows = torch.cat([torch.arange(0, 32), torch.arange(r0 // 32 * 32 - 32, r0 // 32 * 32 + 64), torch.arange(N - 33, N)])
    sub = pos[rows.cuda()].cpu()
    plan = X.plan_of(sub, scale, shift, T, "cuda")

    ob, out = guarded((N, C))
    call("psdf_enc_forward", *args, out)
    torch.cuda.synchronize()
    assert guards_intact(ob)
    got = out[rows.cuda()].clone()
    del ob, out
    gob, g_out = guarded((N, C), 0.0)
    g_out.normal_(generator=g)
    go_sub = g_out[rows.cuda()].cpu()
    ref = X.reference(plan, lat, win, True, 0.5, go_sub, gg[rows.cuda()].cpu(), sub)
    check_dense("forward > 2^31", None, got, ref["out"], ref["A_out"], X.EPS_FWD)
    pb, g_p = guarded((N, D))
    call("psdf_enc_backward", *args, g_out, None, g_p)
    check_dense("pos > 2^31", pb, g_p[rows.cuda()], ref["pos_grad"], ref["A_pos"], X.EPS_POS)
    assert bool(torch.isfinite(g_p).all())
    ggb, g_go = guarded((N, C))
    call("psdf_enc_double_backward", *args, gg, g_out, None, g_go)
    torch.cuda.synchronize()
    assert guards_intact(ggb)
    check_dense("grad_out > 2^31", None, g_go[rows.cuda()], ref["ggo"], ref["A_ggo"], X.EPS_GGO)


def test_table_of_2_31_minus_1_rows(cuda):
    """one level, F = 1, T = 2^31 - 1 (8 GB per table): the backward reaches exactly the oracle's rows, many above 2^30, with the
    reference values; the forward and positions gradient read them. Needs ~18 GB of free device memory."""
    from permuto_sdf_b200 import call
    D, F, L, T, N = 3, 1, 1, 2 ** 31 - 1, 4097
    need = 2 * T * 4 + (4 << 30)
    if _free_bytes() < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 2 ** 30, _free_bytes() / 2 ** 30))
    g = torch.Generator().manual_seed(9)
    pos = torch.rand(N, D, generator=g) * 40 - 20
    scale = eo.scale_factor([1.0], D)
    shift = torch.randn(L, D, generator=g) * 10
    plan = X.plan_of(pos, scale, shift, T, "cuda")
    idx = plan.idx[0].reshape(-1)
    assert int((idx >= 2 ** 30).sum()) > N
    lat = torch.empty(L, T, F, device="cuda")
    lat.view(-1)[idx] = torch.rand(idx.numel(), generator=g).cuda() * 2 - 1
    uniq, inv = torch.unique(idx, return_inverse=True)
    g_out = torch.randn(N, F, generator=g)
    # the reference reads only the hashed rows: hand it those, renumbered
    plan.idx[0], plan.T = inv.view(N, D + 1), uniq.numel()
    ref = X.reference(plan, lat.view(-1)[uniq].view(1, -1, 1), None, False, 1.0, g_out, None, pos)
    args = (N, D, L, F, T, pos.cuda(), lat, scale.cuda(), shift.cuda(), None, 0, 1.0)
    out = torch.empty(N, F, device="cuda")
    call("psdf_enc_forward", *args, out)
    check_dense("forward T=2^31-1", None, out, ref["out"], ref["A_out"], X.EPS_FWD)
    g_l = torch.zeros(L, T, F, device="cuda")
    g_p = torch.empty(N, D, device="cuda")
    call("psdf_enc_backward", *args, g_out.cuda(), g_l, g_p)
    check_dense("pos T=2^31-1", None, g_p, ref["pos_grad"], ref["A_pos"], X.EPS_POS)
    nz = int((g_l.view(-1) != 0).sum())
    assert nz == int((ref["lat_A"].view(-1) > 0).sum()), "the backward touched rows the oracle does not hash to"
    got = g_l.view(-1)[uniq].double()
    bound = X.lattice_bound(ref["lat"].view(-1), ref["lat_A"].view(-1), ref["lat_n"].reshape(-1), None, X.M_LAT)
    w = X.worst((got - ref["lat"].view(-1)).abs(), bound)
    print("  lattice T=2^31-1       worst err/bound %.3f, %d rows above 2^30" % (w, int((uniq >= 2 ** 30).sum())))
    assert w <= 1.0


# ------------------------------------------------------------------------------------------------ autograd wiring
def tiny_head_loss(enc_fn, p, Wm, proj):
    p = p.clone().requires_grad_(True)
    feat = enc_fn(p)
    y = torch.tanh(feat @ Wm).sum(1, keepdim=True)
    (gp,) = torch.autograd.grad(y, p, torch.ones_like(y), create_graph=True)
    loss = (y ** 2).mean() + ((gp.norm(dim=1) - 1.0) ** 2).mean() + (gp * proj).sum(1).mean()
    return gp, loss


@pytest.mark.parametrize("mode", ["float", "deterministic", "grad_in_place"])
@pytest.mark.parametrize("D,F", [(3, 2), (5, 4), (2, 8)])
def test_autograd_wiring(cuda, D, F, mode):
    """PermutoEncoding under create_graph (the eikonal pattern): the positions gradient and the lattice gradient (value path plus
    double backward, accumulated onto a prefilled .grad) against fp64 autograd of the straight-through reference, per element. The
    upstream gradients come from fp32 torch ops (tanh, a product of C terms) whose own rounding is bounded by 2^-16 of their terms, so
    the bound is 2^-12 A with A the reference's error scale at the absolute upstream gradients."""
    import permutohedral_encoding as pe
    L, T, N = 7, 4099, 2000
    torch.manual_seed(D * 10 + F)
    enc = pe.PermutoEncoding(D, T, L, F, np.geomspace(1.0, 1e-3, num=L), concat_points=True, concat_points_scaling=0.5, init_scale=0.3,
                             deterministic=(mode == "deterministic"))
    enc.grad_in_place = mode == "grad_in_place"
    C = enc.output_dims()
    pos = torch.rand(N, D) - 0.5
    win = eo.coarse2fine(L, 0.6)
    Wm, proj = torch.randn(C, 5) * 0.5, torch.randn(N, D)
    pre = torch.randn(L, T, F, device="cuda")
    enc.lattice_values.grad = pre.clone()
    gp, loss = tiny_head_loss(lambda p: enc(p, win.cuda()), pos.cuda(), Wm.cuda(), proj.cuda())
    loss.backward()
    got_l = enc.lattice_values.grad.detach()

    sc, sh = enc.scale_factor.cpu(), enc.shift_tensor().cpu()
    plan = X.plan_of(pos, sc, sh, T, "cuda")
    lat64 = enc.lattice_values.detach().double().requires_grad_(True)
    Wd, projd = Wm.double().cuda(), proj.double().cuda()
    p = pos.double().cuda().requires_grad_(True)
    feat = X.encode_st(p, lat64, plan, win, F, True, 0.5)
    feat.retain_grad()
    z = feat @ Wd
    y = torch.tanh(z).sum(1, keepdim=True)
    (rgp,) = torch.autograd.grad(y, p, torch.ones_like(y), create_graph=True)
    rloss = (y ** 2).mean() + ((rgp.norm(dim=1) - 1.0) ** 2).mean() + (rgp * projd).sum(1).mean()
    rl, rgg = torch.autograd.grad(rloss, (lat64, rgp), retain_graph=True)
    # error scales: the positions gradient at g1 = d y / d feat; the lattice gradient at the value path's upstream and the double
    # backward's (gg = d loss / d gp, g1)
    g1 = torch.autograd.grad(y.sum(), feat, retain_graph=True)[0].detach()
    g0 = torch.autograd.grad(rloss, feat, retain_graph=True)[0].detach()
    a1 = X.reference(plan, enc.lattice_values.detach(), win, True, 0.5, g1.abs(), None, pos)
    a0 = X.reference(plan, enc.lattice_values.detach(), win, True, 0.5, g0.abs(), rgg.detach().abs(), pos)
    a2 = X.reference(plan, enc.lattice_values.detach(), win, True, 0.5, g1.abs(), rgg.detach().abs(), pos)
    eps = 2.0 ** -12
    wp = X.worst((gp.detach().double() - rgp.detach()).abs(), eps * a1["A_pos"])
    A_l = a0["lat_A"] + a2["dlat_A"] + pre.double().abs() * 2.0 ** -12 / eps
    wl = X.worst((got_l.double() - (pre.double() + rl)).abs(), eps * A_l)
    untouched = a0["lat_n"] == 0
    print("\n  autograd %s D=%d F=%d: pos worst %.3f, lattice worst %.3f" % (mode, D, F, wp, wl))
    assert wp <= 1.0 and wl <= 1.0
    assert torch.equal(got_l[untouched], pre[untouched])
