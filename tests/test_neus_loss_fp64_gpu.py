"""The NeuS loss head (csrc/neus_fused.cu: the seven psdf_neus_* entry points) and psdf_loss_terms (csrc/iter_glue.cu) against the fp64
reference of oracle/neus_fp64.py, element by element, at the ray lengths around the 32-sample chunks, at saturated and near-zero alpha,
at every subgradient kink placed exactly, with every NULL combination of the colour head's calibration, with and without background,
curvature, device-side counts and tail rows, in float-atomic and deterministic mode. The C ABI is driven directly, so NULL arguments and
pre-filled buffers are under the test's control.

Bounds, per output tensor:
  * max|got - ref| / max|ref| <= 1e-3;
  * per element |got_i - ref_i| <= EPS A_i (+ n_i 2^-35 in deterministic mode, + one rounding of a pre-filled += buffer), A the error
    scale of oracle/neus_fp64.py (linearised propagation of absolute rounding terms, __expf at its documented bound), EPS = 2^-22;
  * "=" outputs carry NaN-sentinel guard rows past N and R, and rows of skipped rays, which must stay untouched; the tail rows
    [nr_valid, n_rows) must be exactly zero.
The backward reference is evaluated at the forward values the backward reads (see oracle/neus_fp64.py). `pytest -s` prints the error
and the worst element ratio of every case and output."""
import pytest
import torch

from oracle import neus_fp64 as R
from test_fused_backward_fp64_gpu import mode
from test_fused_forward_fp64_gpu import SENTINEL, guarded, rows

pytestmark = pytest.mark.gpu
EPS = R.EPS
FX = 2.0 ** -35
K_DET_IMAGES = 1 << 16
REPORT = []


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\n%-46s %-10s %-9s %12s %12s" % ("case", "kernel", "output", "max rel", "worst ratio"))
        for r in REPORT:
            print("%-46s %-10s %-9s %12.3e %12.3e" % r)
        worst = {}
        for _, k, o, _, w in REPORT:
            worst[(k, o)] = max(worst.get((k, o), 0.0), w)
        print("\nworst element ratio per kernel and output")
        for (k, o), w in sorted(worst.items()):
            print("%-10s %-9s %12.3e" % (k, o, w))


def check(case, kernel, name, got, ref, A, budget=0.0, mask=None, block=True):
    got, ref, A = got.double().cpu().reshape(ref.shape), ref.detach().double().cpu(), A.detach().double().cpu().reshape(ref.shape)
    if mask is not None:
        got, ref, A = got[mask], ref[mask], A[mask]
        if isinstance(budget, torch.Tensor):
            budget = budget[mask]
    err = (got - ref).abs()
    bound = EPS * A + budget
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    mref = float(ref.abs().max()) if ref.numel() else 0.0
    # a tensor whose largest element is this close to fp32's subnormal range cannot be resolved to 1e-3 of it
    block = block and mref >= 2.0 ** -100
    emax = float(err.max()) if err.numel() else 0.0
    blk = emax / mref if mref > 0 else emax
    worst = float(ratio.max()) if ratio.numel() else 0.0
    REPORT.append((case, kernel, name, blk, worst))
    extra = float(torch.as_tensor(budget).max()) if ref.numel() else 0.0
    assert not block or blk <= 1e-3 + extra / max(mref, 1e-300), (case, kernel, name, "block", blk)
    if worst > 1.0:
        i = int(ratio.reshape(-1).argmax())
        raise AssertionError((case, kernel, name, "element", i, "got", float(got.reshape(-1)[i]), "ref", float(ref.reshape(-1)[i]),
                              "A", float(A.reshape(-1)[i]), "ratio", worst, "over", int((ratio > 1).sum())))


def untouched(buf, keep, what):
    """rows `keep` (bool [n]) of a guarded buffer still hold the sentinel"""
    b = buf.cpu()
    if bool(keep.any()):
        assert bool((b[:keep.shape[0]][keep].view(torch.int32) == SENTINEL).all()), (what, "wrote rows of skipped rays")


def rows_of(buf, n, written, what):
    """rows [0, n) of a guarded buffer: the guard rows and the rows not in `written` untouched, the written rows finite"""
    b = buf.cpu()
    assert bool((b[n:].view(torch.int32) == SENTINEL).all()), (what, "written past the end")
    untouched(buf, ~written, what)
    assert bool(torch.isfinite(b[:n][written]).all()), (what, "non-finite rows")
    return b[:n]


# ------------------------------------------------------------------------------------------------ scenes
SPECIAL = [0, 1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 200]


def ray_lengths(R_, g):
    if R_ <= len(SPECIAL):
        return [SPECIAL[(3 * i + 5) % len(SPECIAL)] for i in range(R_)]
    extra = torch.randint(1, 97, (R_ - len(SPECIAL),), generator=g).tolist()
    return SPECIAL + extra


def scene(layout, R_, inv_s, cos_anneal, seed, head=True, bg=False, mask=True, curv=False, cal="full", n_img=5, big_img=False,
          tail=0, skip_rays=1):
    """a packed sample set: ragged (the SPECIAL lengths, then random ones; `skip_rays` rays past max_nr_samples) or equal (fixed_n);
    sdf profiles crossing the surface (saturated alpha at large inv_s), flat far ones (alpha ~ 0), and exactly placed kinks"""
    g = torch.Generator().manual_seed(seed)
    if layout.startswith("equal"):
        fixed_n = int(layout[5:])
        lens = [fixed_n] * R_
        se = torch.zeros(R_, 2, dtype=torch.int32)
        equal = True
    else:
        fixed_n = 0
        lens = ray_lengths(R_, g)
        equal = False
    starts = torch.tensor([0] + lens[:-1]).cumsum(0)
    N = int(sum(lens))
    max_nr = N
    if not equal:
        se = torch.stack([starts, starts + torch.tensor(lens)], 1).to(torch.int32)
        # rays that end past max_nr_samples (their samples are never read): the last ones, re-pointed across the end
        for k in range(min(skip_rays, R_ - 1)):
            i = R_ - 1 - k
            if lens[i] > 0:
                se[i, 0], se[i, 1] = max_nr - 1, max_nr + 5
    dt = torch.zeros(N)
    sdf = torch.zeros(N)
    kind = torch.randint(0, 4, (R_,), generator=g)
    for i, n in enumerate(lens):
        s0 = int(starts[i])
        if n == 0:
            continue
        step = float(torch.rand(1, generator=g)) * 0.02 + 0.004
        t = torch.arange(n, dtype=torch.float32) * step
        dt[s0:s0 + n] = step * (0.5 + torch.rand(n, generator=g))
        k = int(kind[i])
        if k == 3:       # far from the surface: alpha ~ 0
            sdf[s0:s0 + n] = 0.3 + 0.01 * torch.rand(n, generator=g)
        else:            # crossing the surface mid-ray
            sdf[s0:s0 + n] = (t[n // 2] - t) * (0.5 + 0.5 * k) + 1e-3 * torch.randn(n, generator=g)
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1)
    nrm = 0.5 + torch.rand(N, 1, generator=g)
    grad = -dirs * nrm * 0.8 + 0.3 * torch.randn(N, 3, generator=g)
    # kinks: dir (1, 0, 0) and grad (c, y, z) give true_cos = c exactly
    i = torch.arange(N)
    for r, c in ((0, -1.0), (1, 0.0), (2, 1.0)):
        sel = i % 17 == 3 + 4 * r
        dirs[sel] = torch.tensor([1.0, 0.0, 0.0])
        grad[sel, 0] = c
    grad[i % 29 == 7] = 0.0                                                       # |g| = 0
    grad[i % 31 == 11] = torch.nn.functional.normalize(grad[i % 31 == 11] + 1e-3, dim=1) * 1e-13      # |g| < 1e-12
    rgb = torch.randn(N, 3, generator=g) * 2 if head else torch.rand(N, 3, generator=g)
    gt = torch.rand(R_, 3, generator=g)
    hit = (torch.rand(R_, generator=g) > 0.2).to(torch.uint8)
    gm = None
    if mask:
        gm = torch.rand(R_, generator=g)
        gm[torch.arange(R_) % 3 == 0] = 0.0
        gm[torch.arange(R_) % 3 == 1] = 1.0
    bg_rgb = torch.rand(R_, 3, generator=g) if bg else None
    img = wd = bias = None
    fixed = -1
    if head and cal != "none":
        img = torch.randint(0, n_img, (R_,), generator=g).to(torch.int32)
        nw = K_DET_IMAGES + 1 if big_img else n_img
        if big_img:
            img[torch.arange(R_) % 4 == 1] = K_DET_IMAGES
        wd = torch.randn(nw, 3, generator=g) * 0.2 if "wd" in cal or cal == "full" else None
        bias = torch.randn(nw, 3, generator=g) * 0.2 if "b" in cal or cal == "full" else None
        img = img if ("img" in cal or cal == "full") else None
        fixed = 0
    gs = None
    if curv:
        gs = grad + 0.4 * torch.randn(N, 3, generator=g)
        gs[i % 23 == 2] = grad[i % 23 == 2] * 3.0                                 # parallel: dot = 1, in the clamp
        gs[i % 23 == 9] = -grad[i % 23 == 9]                                      # antiparallel
        gs[i % 37 == 5] = 1e-13 * torch.tensor([0.3, -0.5, 0.8])
    return R.NeusInputs(se, R_, N + tail, max_nr, sdf, grad, rgb, dirs, dt, torch.tensor([float(inv_s)]), cos_anneal, gt, gm, hit, bg_rgb,
                        head, img, wd, bias, fixed, gs, equal, fixed_n)


def pad_rows(t, extra):
    """sample tensors with `extra` rows past the rays (the tail of a static-capacity container)"""
    return torch.cat([t, torch.zeros((extra,) + tuple(t.shape[1:]), dtype=t.dtype)]) if extra else t


def cu(t):
    return None if t is None else t.contiguous().cuda()


def rsp(I):
    return (I.R, I.max_nr_samples, cu(I.start_end), int(I.equal), I.fixed_n)


# ------------------------------------------------------------------------------------------------ runs
def run_forward(I, kind, cos_dev=False, N=None):
    """one of the three loss forwards -> dict of rows (guards checked)"""
    from permuto_sdf_b200._lib import call
    N = N or I.sdf.shape[0]
    al, T, w = guarded(N, 0), guarded(N, 0), guarded(N, 0)
    pred, ws, bgT, rl = guarded(I.R, 3), guarded(I.R, 0), guarded(I.R, 0), guarded(I.R, 3)
    cd = torch.tensor([float(I.cos_anneal)], device="cuda") if cos_dev else None
    ca = 0.55 if cos_dev else float(I.cos_anneal)                   # overridden by the device value
    common = (*rsp(I), cu(I.sdf), cu(I.grad), cu(I.rgb), cu(I.dirs), cu(I.dt), cu(I.inv_s), ca, cd, cu(I.gt_rgb), cu(I.gt_mask), cu(I.hit))
    if kind == "render":
        call("psdf_neus_render_loss_forward", *common, cu(I.bg_rgb), al, T, w, pred, ws, bgT, rl)
    elif kind == "head":
        call("psdf_neus_head_loss_forward", *common, cu(I.img_idx), cu(I.weight_delta), cu(I.bias), I.fixed_img, al, T, w, pred, ws, bgT, rl)
    else:
        call("psdf_neus_head_bg_loss_forward", *common, cu(I.img_idx), cu(I.weight_delta), cu(I.bias), I.fixed_img, cu(I.bg_rgb), al, T, w,
             pred, ws, bgT, rl)
    torch.cuda.synchronize()
    return dict(alpha=al, T=T, w=w, pred=pred, wsum=ws, bgT=bgT, ray_loss=rl)


def fwd_rows(out, I, written):
    N = I.sdf.shape[0]
    res = {k: rows_of(out[k], N, written, k) for k in ("alpha", "T", "w")}
    res.update({k: rows(out[k], I.R, k) for k in ("pred", "wsum", "bgT", "ray_loss")})
    return res


def check_forward(case, kernel, I, got):
    ref = R.forward_reference(I)
    A = R.error_scales(I)
    m = ref["rows"]
    # below the clip (s = 1e-6) alpha ~ 1e-5 / (pc + 1e-5) with pc ~ nc ~ 1/2, where __expf's 2 ulp at x ~ 0 are ~1% of alpha: every
    # element stays inside its error scale, the tensor as a whole is not resolved to 1e-3
    resolved = float(I.inv_s.reshape(-1)[0]) >= 1e-6
    for k in ("alpha", "T", "w"):
        check(case, kernel, k, got[k], ref[k], A["A_" + k], mask=m, block=resolved)
    check(case, kernel, "pred", got["pred"], ref["pred"], A["A_pred"])
    check(case, kernel, "wsum", got["wsum"], ref["wsum"], A["A_wsum"])
    check(case, kernel, "bgT", got["bgT"], ref["bgT"], A["A_bgT"])
    check(case, kernel, "ray_loss", got["ray_loss"], ref["ray_loss"], A["A_ray_loss"])
    return ref


def set_gt_to_pred(I, pred):
    """gt of some channels set bit for bit to the kernel's own pred (the L1 sign at 0)"""
    sel = torch.arange(I.R) % 5 == 2
    I.gt_rgb = I.gt_rgb.clone()
    I.gt_rgb[sel, 1] = pred[sel, 1]
    I.gt_rgb[torch.arange(I.R) % 7 == 4] = pred[torch.arange(I.R) % 7 == 4]


# ------------------------------------------------------------------------------------------------ the basic pair
RENDER_CASES = [("ragged", 12, 20.0, 0.37, False), ("ragged", 12, 2981.0, 0.0, True), ("ragged", 9, 512.0, 1.0, False),
                ("ragged", 1, 20.0, 0.37, False), ("ragged", 7, 2981.0, 1.0, True), ("ragged", 8, 1e6, 0.37, False),
                ("ragged", 2000, 2981.0, 0.37, True), ("ragged", 3000, 20.0, 0.0, False), ("equal1", 9, 512.0, 0.37, True),
                ("equal32", 300, 2981.0, 0.37, False), ("equal33", 8, 20.0, 1.0, True), ("equal96", 300, 2981.0, 0.0, True),
                ("ragged", 12, 2e6, 0.37, True), ("ragged", 12, 1e-7, 0.37, False)]


@pytest.mark.parametrize("m", ["float", "det"])
@pytest.mark.parametrize("layout,R_,inv_s,ca,bg", RENDER_CASES, ids=["%s-R%d-s%g-r%g-%s" % (c[:4] + ("bg" if c[4] else "nobg",))
                                                                     for c in RENDER_CASES])
def test_render_loss_pair(cuda, layout, R_, inv_s, ca, bg, m):
    """psdf_neus_render_loss_forward / _backward: g_inv_s pre-filled (+=, gated outside [1e-6, 1e6]), g_total_dev, cos_anneal_dev"""
    from permuto_sdf_b200._lib import call
    I = scene(layout, R_, inv_s, ca, seed=R_ * 7 + int(ca * 10) + (1 if bg else 0), head=False, bg=bg, mask=(R_ % 2 == 0))
    case = "%s R%d s%g r%g%s %s" % (layout, R_, inv_s, ca, " bg" if bg else "", m)
    cos_dev = R_ % 3 == 0
    with mode(m, 1 << 16):
        out = run_forward(I, "render", cos_dev)
        probe = R.forward_reference(I)
        got = fwd_rows(out, I, probe["rows"])
        set_gt_to_pred(I, got["pred"])
        out = run_forward(I, "render", cos_dev)
        got = fwd_rows(out, I, probe["rows"])
        ref = check_forward(case, "render", I, got)
        N = I.sdf.shape[0]
        gsdf, ggrad, grgb, gbg = guarded(N, 0), guarded(N, 3), guarded(N, 3), guarded(I.R, 3)
        init = torch.tensor([0.25], device="cuda")
        ginv = init.clone()
        gtot = torch.tensor([1.7], device="cuda")
        sr, sm, se = 1.0 / (3 * I.R), 0.3 / I.R, 0.1 / max(N, 1)
        cd = torch.tensor([float(ca)], device="cuda") if cos_dev else None
        call("psdf_neus_render_loss_backward", *rsp(I), cu(I.sdf), cu(I.grad), cu(I.rgb), cu(I.dirs), cu(I.dt), cu(I.inv_s),
             0.55 if cos_dev else ca, cd, cu(I.gt_rgb), cu(I.gt_mask), cu(I.hit), cu(I.bg_rgb), out["alpha"], out["T"], out["pred"],
             out["wsum"], out["bgT"], gtot, sr, sm, se, None, gsdf, ggrad, grgb, gbg if bg else None, ginv)
        torch.cuda.synchronize()
        g1 = gsdf.clone()
        if m == "det":       # two runs give the same bits
            ginv2 = init.clone()
            call("psdf_neus_render_loss_backward", *rsp(I), cu(I.sdf), cu(I.grad), cu(I.rgb), cu(I.dirs), cu(I.dt), cu(I.inv_s),
                 0.55 if cos_dev else ca, cd, cu(I.gt_rgb), cu(I.gt_mask), cu(I.hit), cu(I.bg_rgb), out["alpha"], out["T"], out["pred"],
                 out["wsum"], out["bgT"], gtot, sr, sm, se, None, gsdf, ggrad, grgb, gbg if bg else None, ginv2)
            torch.cuda.synchronize()
            assert torch.equal(ginv, ginv2) and torch.equal(g1.view(torch.int32), gsdf.view(torch.int32))
    saved = dict(alpha=got["alpha"], pred=got["pred"], wsum=got["wsum"], bgT=got["bgT"])
    ref = R.backward_reference(I, saved, sr, sm, se, 0.0, 1.7)
    A = R.error_scales(I, saved, sr, sm, se, 0.0, 1.7)
    w = ref["rows"]
    resolved = 1e-6 <= inv_s                    # see check_forward
    check(case, "render", "g_sdf", rows_of(gsdf, N, w, "g_sdf"), ref["sdf"], A["A_sdf"], mask=w, block=resolved)
    check(case, "render", "g_grad", rows_of(ggrad, N, w, "g_grad"), ref["grad"], A["A_grad"], mask=w)
    check(case, "render", "g_rgb", rows_of(grgb, N, w, "g_rgb"), ref["rgb"], A["A_rgb"], mask=w)
    if bg:
        check(case, "render", "g_bg_rgb", rows(gbg, I.R, "g_bg_rgb"), ref["bg_rgb"], A["A_bg_rgb"])
    g_inv = ginv.cpu().double() - 0.25
    if not (1e-6 <= inv_s <= 1e6):
        assert float(ginv) == 0.25, ("g_inv_s changed outside the clip", float(ginv))
    else:
        nray = float((~R.Layout(I.start_end, I.R, I.max_nr_samples, I.equal, I.fixed_n).skip).sum())
        # deterministic: one 2^-35 rounding per ray, one flush into the pre-filled value; float atomics: every ray's add rounds the
        # running total, pre-filled value included
        budget = (nray + 1) * FX + 2 * float(ginv.abs()) * 2.0 ** -24 if m == "det" else (nray + 1) * float(ginv.abs()) * 2.0 ** -24
        check(case, "render", "g_inv_s", g_inv, ref["inv_s"], A["A_inv_s"], budget=budget)


# ------------------------------------------------------------------------------------------------ head variants
HEAD_CASES = [
    # layout, R, inv_s, cos_anneal, bg, cal, big_img, curv, tail
    ("ragged", 12, 2981.0, 0.37, False, "full", False, True, 40),
    ("ragged", 12, 20.0, 0.0, True, "full", False, True, 0),
    ("ragged", 9, 512.0, 1.0, False, "none", False, False, 0),
    ("ragged", 8, 2981.0, 0.37, True, "img+wd", False, True, 7),
    ("ragged", 7, 20.0, 0.37, False, "img+b", False, False, 0),
    ("ragged", 12, 512.0, 0.37, False, "wd+b", False, True, 0),
    ("ragged", 2000, 2981.0, 0.37, True, "full", True, True, 300),
    ("ragged", 1500, 512.0, 0.0, False, "full", True, False, 0),
    ("equal1", 9, 20.0, 0.37, False, "full", False, True, 5),
    ("equal32", 257, 2981.0, 1.0, True, "full", False, True, 0),
    ("equal33", 8, 512.0, 0.37, False, "img+wd", False, False, 3),
    ("equal96", 300, 2981.0, 0.37, True, "full", False, True, 64),
]


@pytest.mark.parametrize("m", ["float", "det"])
@pytest.mark.parametrize("layout,R_,inv_s,ca,bg,cal,big,curv,tail", HEAD_CASES,
                         ids=["%s-R%d-s%g-r%g-%s-%s%s%s-t%d" % (c[:4] + ("bg" if c[4] else "nobg", c[5], "-big" if c[6] else "",
                                                                          "-curv" if c[7] else "", c[8])) for c in HEAD_CASES])
def test_head_loss_pair(cuda, layout, R_, inv_s, ca, bg, cal, big, curv, tail, m):
    """psdf_neus_head_loss_* / _head_bg_loss_*: calibration NULL combinations and fixed_img, an image index >= kDetImages, curvature with
    curv_scale_dev and nr_samples_dev, the tail rows [nr_valid, n_rows), g_weight_delta / g_bias pre-filled (+=)"""
    from permuto_sdf_b200._lib import call
    I = scene(layout, R_, inv_s, ca, seed=1000 + R_ + tail, head=True, bg=bg, mask=True, curv=curv, cal=cal, big_img=big)
    kind = "head_bg" if bg else "head"
    case = "%s R%d s%g r%g %s%s t%d %s" % (layout, R_, inv_s, ca, cal, " curv" if curv else "", tail, m)
    N = I.sdf.shape[0]
    with mode(m, 1 << 16):
        probe = R.forward_reference(I)
        got = fwd_rows(run_forward(I, kind, cos_dev=R_ % 2 == 1), I, probe["rows"])
        set_gt_to_pred(I, got["pred"])
        out = run_forward(I, kind, cos_dev=R_ % 2 == 1)
        got = fwd_rows(out, I, probe["rows"])
        check_forward(case, kind, I, got)
        # the render mode: bit for bit the training forward's pred and w_sum, normals and the background term against the reference
        if R_ % 2 == 0 or bg:
            pr, pb, nm, wr = guarded(I.R, 3), guarded(I.R, 3), guarded(I.R, 3), guarded(I.R, 0)
            call("psdf_neus_render_forward", *rsp(I), cu(I.sdf), cu(I.grad), cu(I.rgb), cu(I.dirs), cu(I.dt), cu(I.inv_s), float(I.cos_anneal),
                 cu(I.img_idx), cu(I.weight_delta), cu(I.bias), I.fixed_img, cu(I.bg_rgb), pr, pb if bg else None, nm, wr)
            torch.cuda.synchronize()
            assert torch.equal(rows(pr, I.R, "pred"), got["pred"]) and torch.equal(rows(wr, I.R, "wsum"), got["wsum"])
            A = R.error_scales(I)
            check(case, "render_fwd", "normals", rows(nm, I.R, "normals"), probe["normals"], A["A_normals"])
            if bg:
                check(case, "render_fwd", "pred_bg", rows(pb, I.R, "pred_bg"), probe["pred_bg"], A["A_pred_bg"])
            else:
                assert bool((pb.cpu().view(torch.int32) == SENTINEL).all())
        # backward: n_rows = N + tail rows, nr_valid_dev = N; nr_samples_dev = N + 3 (the mean's divisor); curv_scale_dev
        n_rows = N + tail
        nv = torch.tensor([N], dtype=torch.int32, device="cuda") if tail else None
        nsd = torch.tensor([N + 3], dtype=torch.int32, device="cuda") if R_ % 2 == 0 else None
        csd = torch.tensor([0.6], device="cuda") if curv else None
        gsdf, ggrad, gx, ggs = guarded(n_rows, 0), guarded(n_rows, 3), guarded(n_rows, 3), guarded(n_rows, 3) if curv else None
        gbg = guarded(I.R, 3) if bg else None
        nimg = I.weight_delta.shape[0] if I.weight_delta is not None else 5
        init_w = torch.randn(nimg, 3, generator=torch.Generator().manual_seed(3)).cuda()
        gwd, gb = init_w.clone(), (init_w * 0.5).clone()
        sr, sm, se, ck = 1.0 / (3 * I.R), 0.3 / I.R, 0.1, 0.05
        grad_s = cu(pad_rows(I.gs, tail)) if curv else None
        pad = lambda t: cu(pad_rows(t, tail))
        args = (*rsp(I), pad(I.sdf), pad(I.grad), pad(I.rgb), pad(I.dirs), pad(I.dt), cu(I.inv_s), 0.55 if R_ % 2 == 1 else ca,
                torch.tensor([float(ca)], device="cuda") if R_ % 2 == 1 else None, cu(I.gt_rgb), cu(I.gt_mask), cu(I.hit), cu(I.img_idx),
                cu(I.weight_delta), cu(I.bias), I.fixed_img)
        saved_b = (out["alpha"], out["T"], out["pred"], out["wsum"], out["bgT"], sr, sm, se if nsd is not None else se / N, nsd, grad_s, ck,
                   csd, n_rows, nv, gsdf, ggrad, gx, ggs)
        if bg:
            call("psdf_neus_head_bg_loss_backward", *args, cu(I.bg_rgb), *saved_b, gbg, gwd, gb)
        else:
            call("psdf_neus_head_loss_backward", *args, *saved_b, gwd, gb)
        torch.cuda.synchronize()
        if m == "det":
            gwd2, gb2 = init_w.clone(), (init_w * 0.5).clone()
            if bg:
                call("psdf_neus_head_bg_loss_backward", *args, cu(I.bg_rgb), *saved_b, gbg, gwd2, gb2)
            else:
                call("psdf_neus_head_loss_backward", *args, *saved_b, gwd2, gb2)
            torch.cuda.synchronize()
            assert torch.equal(gwd, gwd2) and torch.equal(gb, gb2), "deterministic mode: two runs differ"
    saved = dict(alpha=got["alpha"], pred=got["pred"], wsum=got["wsum"], bgT=got["bgT"])
    cnt = (N + 3) if nsd is not None else max(I.max_nr_samples, 1)
    sei = se / (N + 3) if nsd is not None else se / N
    ckk = ck * (0.6 if curv else 1.0) / cnt
    ref = R.backward_reference(I, saved, sr, sm, sei, ckk)
    A = R.error_scales(I, saved, sr, sm, sei, ckk)
    w = ref["rows"]
    wn = torch.cat([w, torch.ones(tail, dtype=torch.bool)])
    for nm_, buf, key in (("g_sdf", gsdf, "sdf"), ("g_grad", ggrad, "grad"), ("g_x", gx, "rgb")) + ((("g_gs", ggs, "gs"),) if curv else ()):
        b = rows_of(buf, n_rows, wn if tail else w, nm_)
        assert bool((b[N:n_rows] == 0).all()), (case, nm_, "tail rows [nr_valid, n_rows) not zero")
        key_A = {"sdf": "A_sdf", "grad": "A_grad", "rgb": "A_rgb", "gs": "A_gs"}[key]
        check(case, kind, nm_, b[:N], ref[key], A[key_A], mask=w)
    if bg:
        check(case, kind, "g_bg_rgb", rows(gbg, I.R, "g_bg_rgb"), ref["bg_rgb"], A["A_bg_rgb"])
    if "wd" in ref:
        nper = torch.zeros(nimg, 3, dtype=torch.float64)
        lay = R.Layout(I.start_end, I.R, I.max_nr_samples, I.equal, I.fixed_n)
        live = (I.img_idx.long() != I.fixed_img) & ~lay.skip
        nper.index_add_(0, I.img_idx.long()[live], torch.ones(int(live.sum()), 3, dtype=torch.float64))
        det_ok = torch.arange(nimg)[:, None] < K_DET_IMAGES
        budget = torch.where(det_ok, nper * FX, torch.zeros_like(nper)) if m == "det" else torch.zeros_like(nper)
        # float atomics round the running total, pre-filled value included, once per ray of the image; the flush rounds it once
        adds = torch.where(det_ok, torch.full_like(nper, 2.0), nper + 1.0) if m == "det" else nper + 1.0
        slack_w = adds * gwd.cpu().double().abs() * 2.0 ** -24
        check(case, kind, "g_wd", gwd.cpu().double() - init_w.cpu().double(), ref["wd"], A["A_wd"], budget=budget + slack_w)
        if I.bias is not None:
            slack_b = adds * gb.cpu().double().abs() * 2.0 ** -24
            check(case, kind, "g_bias", gb.cpu().double() - 0.5 * init_w.cpu().double(), ref["bias"], A["A_bias"], budget=budget + slack_b)
    elif I.weight_delta is not None or I.img_idx is not None:
        assert torch.equal(gwd, init_w), "calibration gradient without calibration"


# ------------------------------------------------------------------------------------------------ psdf_loss_terms
LT_CASES = [(5000, 300, False, False, True, True), (300, 5000, True, True, True, True), (1, 1, False, False, False, False),
            (70000, 2000, True, True, True, True), (4000, 9, False, True, False, True)]


@pytest.mark.parametrize("m", ["float", "det"])
@pytest.mark.parametrize("N,R_,nvalid,nmean,curv,off", LT_CASES, ids=["N%d-R%d%s%s%s%s" % (c[:2] + tuple(s if f else "" for s, f in
                                                                                      zip(("-nv", "-nm", "-curv", "-off"), c[2:])))
                                                                    for c in LT_CASES])
def test_loss_terms(cuda, N, R_, nvalid, nmean, curv, off, m):
    """several blocks meeting in the last-block ticket; acc left zero and a second launch identical; nr_valid_dev / nr_mean_dev as
    divisors; g_off with exact zeros of sdf_off; the Lipschitz product across softplus' threshold 20"""
    from permuto_sdf_b200._lib import call
    g = torch.Generator().manual_seed(N + R_)
    grad = torch.randn(N, 3, generator=g)
    gs = grad + 0.5 * torch.randn(N, 3, generator=g) if curv else None
    if curv:
        gs[::11] = grad[::11] * 2
        gs[5::13] = -grad[5::13]
        grad[7::17] = 0.0
    rl = torch.rand(R_, 3, generator=g)
    n_off = 777
    so = (torch.rand(n_off, generator=g) - 0.5) * 0.1
    so[::9] = 0.0
    nv = N - N // 7 if nvalid else N
    nm_ = nv // 2 + 3 if nmean else None
    lip = [torch.tensor([x]) for x in (0.5, 25.0, -3.0, 19.999)]
    wcd = torch.tensor([0.7])
    ref = R.loss_terms_reference(N, nv, nm_, grad, gs, R_, rl, so if off else None, 1 / (3 * R_), 0.2 / R_, 0.1, 0.3, 0.7, 0.4, 2e-3, lip)
    acc = torch.zeros(8, device="cuda")
    with mode(m, 1 << 16):
        results = []
        for _ in range(2):
            loss, terms, goff = guarded(1, 0), guarded(12, 0), guarded(n_off, 0)
            call("psdf_loss_terms", N, torch.tensor([nv], dtype=torch.int32, device="cuda") if nvalid else None,
                 torch.tensor([nm_], dtype=torch.int32, device="cuda") if nmean else None, cu(grad), cu(gs), R_, cu(rl), n_off,
                 cu(so) if off else None, goff if off else None, 1 / (3 * R_), 0.2 / R_, 0.1, 0.3, cu(wcd), 0.4, 2e-3, *[cu(c) for c in lip],
                 acc, loss, terms)
            torch.cuda.synchronize()
            assert bool((acc == 0).all()), "acc not left zero"
            results.append((loss.clone(), terms.clone(), goff.clone()))
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(results[0][:2], results[1][:2])) or m == "float"
    loss, terms, goff = results[1]
    case = "loss_terms N%d R%d %s" % (N, R_, m)
    budget = 6 * FX * (N + R_ + n_off) if m == "det" else 0.0
    check(case, "terms", "loss", rows(loss, 1, "loss"), ref["loss"], ref["A_loss"], budget=budget)
    t = rows(terms, 10, "terms")                      # terms [10, 12) are not written
    check(case, "terms", "terms", t, ref["terms"], ref["A_terms"], budget=budget)
    if off:
        check(case, "terms", "g_off", rows(goff, n_off, "g_off"), ref["g_off"], ref["A_g_off"])
    else:
        assert bool((goff.cpu().view(torch.int32) == SENTINEL).all())


# ------------------------------------------------------------------------------------------------ one iteration end to end
@pytest.mark.parametrize("bg,mask,curv", [(False, True, True), (True, False, True), (False, False, False), (True, True, False)],
                         ids=["mask-curv", "bg-curv", "plain", "bg-mask"])
def test_iteration_loss_and_gradients_agree(cuda, bg, mask, curv):
    """forward -> psdf_loss_terms -> backward with the scale arguments built as Iteration builds them (c_rgb = 1/(3R), c_mask = w_mask/R,
    scale_eik = w_eik with the device count, w_curv with its device multiplier): the reported loss is the fp64 total loss, and every
    backward output is d(that loss)/d(input), g_off d(loss)/d sdf_off"""
    from permuto_sdf_b200._lib import call
    I = scene("ragged", 600, 512.0, 0.37, seed=77, head=True, bg=bg, mask=mask, curv=curv, cal="full", skip_rays=0)
    N = I.sdf.shape[0]
    kind = "head_bg" if bg else "head"
    out = run_forward(I, kind, cos_dev=True)
    got = fwd_rows(out, I, R.forward_reference(I)["rows"])
    w_eik, w_mask, w_curv, w_off = 0.04, 0.3 if mask else 0.0, 0.65, 0.2
    c_rgb, c_mask = 1.0 / (3.0 * I.R), w_mask / I.R
    n_valid = torch.tensor([N], dtype=torch.int32, device="cuda")
    wcd = torch.tensor([0.8], device="cuda")
    so = torch.linspace(-0.02, 0.02, 101)
    so[50] = 0.0
    acc, loss, terms, goff = torch.zeros(8, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(12, device="cuda"), guarded(101, 0)
    out_grad = cu(I.grad)
    call("psdf_loss_terms", N, n_valid, None, out_grad, cu(I.gs), I.R, out["ray_loss"], 101, cu(so), goff, c_rgb, c_mask, w_eik,
         w_curv if curv else 0.0, wcd, w_off, 0.0, None, None, None, None, acc, loss, terms)
    gsdf, ggrad, gx, ggs = torch.zeros(N, device="cuda"), torch.zeros(N, 3, device="cuda"), torch.zeros(N, 3, device="cuda"), \
        torch.zeros(N, 3, device="cuda") if curv else None
    gbg = torch.zeros(I.R, 3, device="cuda") if bg else None
    gwd, gb = torch.zeros_like(cu(I.weight_delta)), torch.zeros_like(cu(I.bias))
    args = (*rsp(I), cu(I.sdf), out_grad, cu(I.rgb), cu(I.dirs), cu(I.dt), cu(I.inv_s), 0.0, torch.tensor([float(I.cos_anneal)], device="cuda"),
            cu(I.gt_rgb), cu(I.gt_mask), cu(I.hit), cu(I.img_idx), cu(I.weight_delta), cu(I.bias), I.fixed_img)
    tail = (out["alpha"], out["T"], out["pred"], out["wsum"], out["bgT"], c_rgb, c_mask, w_eik, n_valid, cu(I.gs), w_curv if curv else 0.0,
            wcd, N, n_valid, gsdf, ggrad, gx, ggs)
    if bg:
        call("psdf_neus_head_bg_loss_backward", *args, cu(I.bg_rgb), *tail, gbg, gwd, gb)
    else:
        call("psdf_neus_head_loss_backward", *args, *tail, gwd, gb)
    torch.cuda.synchronize()
    # the fp64 total loss as one function of the inputs (the per-ray terms of the reference, then the loss terms)
    ref = R.forward_reference(I, leaves=True)
    lv = ref["lv"]
    so64 = so.double().requires_grad_(True)
    rl = ref["ray_loss"]
    total = c_rgb * rl[:, 0].sum() + c_mask * rl[:, 1].sum() + w_eik / N * ref["eik"].sum() + w_off * torch.exp(-100.0 * so64.abs()).mean()
    if curv:
        total = total + w_curv * 0.8 * ref["curv"].sum() / N
    A_loss = R.loss_terms_reference(N, N, None, I.grad, I.gs, I.R, rl.detach(), so, c_rgb, c_mask, w_eik, w_curv if curv else 0.0, 0.8,
                                    w_off, 0.0, [])["A_loss"]
    A_f = R.error_scales(I)["A_ray_loss"]
    A_tot = A_loss + (A_f[:, 0].sum() * c_rgb + A_f[:, 1].sum() * c_mask + A_f[:, 2].sum() * w_eik / N)
    check("e2e %s" % kind, "e2e", "loss", loss.cpu(), total.detach().reshape(1), A_tot.reshape(1))
    keys = [k for k in ("sdf", "grad", "rgb", "bg_rgb", "wd", "bias", "gs") if k in lv]
    grads = torch.autograd.grad(total, [lv[k] for k in keys] + [so64], allow_unused=True)
    saved = dict(alpha=got["alpha"], pred=got["pred"], wsum=got["wsum"], bgT=got["bgT"])
    A = R.error_scales(I, saved, c_rgb, c_mask, w_eik / N, w_curv * 0.8 / N if curv else 0.0)
    # d(total)/d(input) at the forward values the backward reads (the kernel's alpha, pred, w_sum, bg_T): a different point than the
    # fp64 forward by the forward's rounding, where the L1 sign and the BCE clip decide as in the kernel; the gradient at the fp64
    # forward agrees per tensor
    at_saved = R.backward_reference(I, saved, c_rgb, c_mask, w_eik / N, w_curv * 0.8 / N if curv else 0.0)
    w = ref["rows"]
    for k, gg in zip(keys, grads):
        gk = {"sdf": gsdf, "grad": ggrad, "rgb": gx, "bg_rgb": gbg, "wd": gwd, "bias": gb, "gs": ggs}[k].cpu().double()
        Ak = A[{"sdf": "A_sdf", "grad": "A_grad", "rgb": "A_rgb", "bg_rgb": "A_bg_rgb", "wd": "A_wd", "bias": "A_bias", "gs": "A_gs"}[k]]
        check("e2e %s" % kind, "e2e", "g_" + k, gk, at_saved[k], Ak, mask=w if k in ("sdf", "grad", "rgb", "gs") else None)
        gref = torch.zeros_like(lv[k]) if gg is None else gg.detach()
        rel = float((gk.reshape(gref.shape) - gref).abs().max()) / max(float(gref.abs().max()), 1e-300)
        REPORT.append(("e2e %s at fp64 forward" % kind, "e2e", "g_" + k, rel, 0.0))
        assert rel <= 1e-3, (k, "against the gradient at the fp64 forward", rel)
    A_goff = R.loss_terms_reference(N, N, None, I.grad, None, I.R, rl.detach(), so, c_rgb, c_mask, w_eik, 0.0, None, w_off, 0.0, [])["A_g_off"]
    check("e2e %s" % kind, "e2e", "g_off", rows(goff, 101, "g_off"), grads[-1], A_goff)
