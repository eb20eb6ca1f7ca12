"""Checks of oracle/neus_fp64.py itself, without a GPU: its forward reproduces the reference project's own outputs (the golden fixture),
its gradients are the derivatives of its loss (gradcheck, away from every kink, where the clamped cumprod backward is the true one), and
EPS A covers an fp32 emulation of the kernels' forward arithmetic (serial transmittance chain, 32-sample chunks, __expf at its
documented error bound)."""
import os

import numpy as np
import pytest
import torch

from oracle import neus_fp64 as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refpy_golden.npz")


@pytest.fixture(scope="module")
def G():
    return np.load(GOLDEN)


@pytest.mark.parametrize("mode", ["free", "forced"])
def test_forward_matches_reference_project(G, mode):
    """weights, weights_sum, bg_transmittance, pred and inv_s of VolumeRenderingNeus on the fixture's ragged set (with an empty ray);
    the fixture's gradients carry the reference kernel's green-channel bug and are not used"""
    t = lambda k: torch.from_numpy(np.array(G[k]))
    se = t("rgb_in.ray_start_end_idx")
    N = G["neus_in.sdf"].shape[0]
    variance = float(G["neus_in.forced"]) if mode == "forced" else 0.3
    inv_s = torch.exp(torch.tensor([variance * 10.0], dtype=torch.float64)).float()
    I = R.NeusInputs(se, se.shape[0], N, N, t("neus_in.sdf").reshape(-1), t("neus_in.gradients"), t("neus_in.rgb"), t("rgb_in.dirs"),
                     t("neus_in.dt").reshape(-1), inv_s, float(G["neus_in.cos_anneal"]))
    ref = R.forward_reference(I)
    A = R.error_scales(I)
    p = "neus_%s." % mode
    assert abs(float(inv_s) - float(G[p + "inv_s"][0])) <= 2e-7 * float(inv_s)
    for name, got, A_, key in (("weights", ref["w"], A["A_w"], "weights"), ("weights_sum", ref["wsum"], A["A_wsum"], "weights_sum"),
                               ("bg_transmittance", ref["bgT"], A["A_bgT"], "bg_transmittance"), ("pred", ref["pred"], A["A_pred"], "pred")):
        want = torch.from_numpy(G[p + key]).double().reshape(got.shape)
        err = (got.detach() - want).abs()
        # the fixture is fp32 torch with libm expf (2 ulp, not __expf's): inside the error scale
        assert float(err.max()) <= 1e-5 * max(float(want.abs().max()), 1e-30), (name, float(err.max()))
        assert bool((err <= R.EPS * A_ + 2.0 ** -24 * want.abs()).all()), (name, float((err / (R.EPS * A_)).max()))
    assert float(ref["bgT"][1]) == 1.0 and float(ref["wsum"][1]) == 0.0          # the empty ray


def small_problem(seed, head, bg, mask, curv):
    g = torch.Generator().manual_seed(seed)
    lens = [5, 1, 0, 7]
    st = torch.tensor([0] + lens[:-1]).cumsum(0)
    se = torch.stack([st, st + torch.tensor(lens)], 1).to(torch.int32)
    N, Rr = sum(lens), len(lens)
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1)
    grad = -dirs * 0.9 + 0.2 * torch.randn(N, 3, generator=g)          # true_cos in (-1, 0): away from the relu kinks
    sdf = torch.linspace(0.05, -0.05, N) + 0.003 * torch.randn(N, generator=g)
    dt = torch.full((N,), 0.02)
    rgb = torch.randn(N, 3, generator=g)
    gt = torch.full((Rr, 3), 5.0)                                       # pred < gt everywhere: the L1 sign is fixed
    gm = torch.tensor([0.0, 1.0, 0.4, 0.7]) if mask else None
    I = R.NeusInputs(se, Rr, N, N, sdf, grad, rgb, dirs, dt, torch.tensor([30.0]), 0.37, gt, gm, None,
                     torch.rand(Rr, 3, generator=g) if bg else None, head, torch.tensor([0, 1, 1, 2], dtype=torch.int32) if head else None,
                     torch.randn(3, 3, generator=g) * 0.1 if head else None, torch.randn(3, 3, generator=g) * 0.1 if head else None, 2,
                     grad + 0.3 * torch.randn(N, 3, generator=g) if curv else None)
    return I


@pytest.mark.parametrize("head,bg,mask,curv", [(False, False, True, False), (True, True, False, True), (True, False, True, True)])
def test_gradients_are_derivatives(head, bg, mask, curv):
    """gradcheck of the whole loss head (custom clamped cumprod included) at a point away from every kink, where max(b, 1e-6) = b"""
    I = small_problem(3, head, bg, mask, curv)
    out0 = R.forward_reference(I)
    fac = 1.0 - out0["alpha_pad"] + 1e-7
    assert bool((fac[out0["layout"].valid] > 1e-6).all())
    live = out0["layout"].valid.any(1)
    assert bool(((out0["wsum"] > 1e-3) & (out0["wsum"] < 1 - 1e-3))[live].all())
    names = ["sdf", "grad", "rgb", "inv_s"] + (["bg_rgb"] if bg else []) + (["weight_delta", "bias"] if head else []) + (["gs"] if curv else [])

    def f(*xs):
        o = _forward_with(I, dict(zip(names, xs)))
        return R.head_loss(o, 0.3, 0.2, 0.1, 0.05 if curv else 0.0, 1.3)

    xs = [getattr(I, n).double().clone().requires_grad_(True) for n in names]
    assert torch.autograd.gradcheck(f, xs, eps=1e-7, atol=1e-6, rtol=1e-5)


def _forward_with(I, xs):
    """forward_reference whose inputs are the given fp64 tensors themselves (gradcheck differentiates through them)"""
    J = R.NeusInputs(**{**I.__dict__})
    for k, v in xs.items():
        setattr(J, k, v)
    orig = R._f64
    try:
        R._f64 = lambda t: None if t is None else (t if t.dtype == torch.float64 else t.detach().double())
        out = R.forward_reference(J, leaves=False)
    finally:
        R._f64 = orig
    return out


def test_clamped_cumprod_backward():
    """the custom backward is the true derivative where 1 - alpha + 1e-7 >= 1e-6, and divides by 1e-6 below"""
    b = torch.tensor([[0.9, 0.5, 1e-5, 0.7, 0.3]], dtype=torch.float64, requires_grad=True)
    valid = torch.ones_like(b, dtype=torch.bool)
    last = torch.zeros_like(valid)
    last[0, -1] = True
    assert torch.autograd.gradcheck(lambda x: R.ClampedCumprod.apply(x, valid, last), (b,))
    b2 = torch.tensor([[0.9, 1e-7, 0.7, 0.3]], dtype=torch.float64, requires_grad=True)
    v2, l2 = torch.ones_like(b2, dtype=torch.bool), torch.tensor([[False, False, False, True]])
    T, bg = R.ClampedCumprod.apply(b2, v2, l2)
    (T.sum() + bg.sum()).backward()
    # d/d b_1 of (T_2 + T_3 + bg) = (T_2 + T_3 + bg) / b_1 on the true path; the clamp divides by 1e-6 instead of 1e-7
    want = float((T[0, 2] + T[0, 3] + bg[0]).detach() / 1e-6)
    assert abs(float(b2.grad[0, 1]) - want) <= 1e-9 * abs(want)


# ------------------------------------------------------------------------------------------------ fp32 emulation of the forward kernel
def _sigmoid_fast32(x, sign):
    """1 / (1 + __expf(-x)) in fp32 with __expf's error at its bound (2 + floor(1.173 |x|) ulp) of the given sign"""
    e = torch.exp(-x.double())
    ulp = 2.0 ** (torch.floor(torch.log2(e.clamp(min=1e-300))) - 23)
    e = (e + sign * (2.0 + torch.floor(1.173 * x.double().abs())) * ulp).float()
    return torch.tensor(1.0, dtype=torch.float32) / (1.0 + e)


def emulate_forward(I, sign):
    """k_neus_forward<false> in fp32: per ray, 32-sample chunks, the serial chain in sample order"""
    lay = R.Layout(I.start_end, I.R, I.max_nr_samples, I.equal, I.fixed_n)
    f = lambda t: lay.gather(t.float())
    sdf, g, d, dt, c = f(I.sdf), f(I.grad), f(I.dirs), f(I.dt), f(I.rgb)
    s = torch.clamp(I.inv_s.float(), 1e-6, 1e6)
    r = torch.tensor(I.cos_anneal, dtype=torch.float32)
    tc = d[..., 0] * g[..., 0] + d[..., 1] * g[..., 1] + d[..., 2] * g[..., 2]
    a = torch.clamp(-tc * 0.5 + 0.5, min=0.0)
    b = torch.clamp(-tc, min=0.0)
    ic = -(a * (1.0 - r) + b * r)
    nxt, prv = sdf + ic * dt * 0.5, sdf - ic * dt * 0.5
    pc, nc = _sigmoid_fast32(prv * s, sign), _sigmoid_fast32(nxt * s, -sign)
    q = (pc - nc + 1e-5) / (pc + 1e-5)
    alpha = torch.where(lay.valid, q.clamp(0.0, 1.0), torch.zeros_like(q))
    T = torch.ones(I.R, dtype=torch.float32)
    Ts, ws, pred = torch.zeros_like(alpha), torch.zeros(I.R), torch.zeros(I.R, 3)
    for k in range(lay.L):
        ak = alpha[:, k]
        Ts[:, k] = T
        wk = ak * T
        pred = pred + wk[:, None] * c[:, k]
        ws = ws + wk
        step = lay.valid[:, k] & ~lay.last[:, k]
        T = torch.where(step, T * (1.0 - ak + 1e-7), T)
    return dict(alpha=alpha, T=Ts, pred=pred, wsum=ws, bgT=T, lay=lay)


@pytest.mark.parametrize("inv_s", [20.0, 512.0, 2981.0])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_error_scale_covers_fp32_emulation(inv_s, sign):
    """the kernels' forward arithmetic, emulated in fp32 with the worst-case __expf error, stays inside EPS A at ray lengths across
    the chunks, at saturated and near-zero alpha"""
    g = torch.Generator().manual_seed(int(inv_s))
    lens = [1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 200, 17]
    st = torch.tensor([0] + lens[:-1]).cumsum(0)
    se = torch.stack([st, st + torch.tensor(lens)], 1).to(torch.int32)
    N = sum(lens)
    sdf = torch.cat([torch.linspace(0.05, -0.05 * (1 + i % 3), n) if i % 4 != 3 else torch.full((n,), 0.3) for i, n in enumerate(lens)])
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1)
    grad = -dirs * 0.9 + 0.3 * torch.randn(N, 3, generator=g)
    dt = 0.005 + 0.01 * torch.rand(N, generator=g)
    I = R.NeusInputs(se, len(lens), N, N, sdf, grad, torch.rand(N, 3, generator=g), dirs, dt, torch.tensor([inv_s]), 0.37)
    ref, A = R.forward_reference(I), R.error_scales(I)
    em = emulate_forward(I, sign)
    lay = em["lay"]
    if inv_s > 1000:
        assert bool((ref["alpha_pad"][lay.valid] == 1.0).any() or (em["alpha"][lay.valid] == 1.0).any())
    worst = 0.0
    for k, key in (("alpha", "alpha"), ("T", "T"), ("w", None)):
        if key is None:
            continue
        got = R.Layout.scatter(lay, em[key].double(), N)[0]
        err = (got - ref[k])[ref["rows"]].abs()
        ratio = float((err / (R.EPS * A["A_" + k][ref["rows"]]).clamp(min=1e-300)).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (k, ratio)
    for k in ("pred", "wsum", "bgT"):
        err = (em[k].double() - ref[k].detach()).abs()
        ratio = float((err / (R.EPS * A["A_" + k]).clamp(min=1e-300)).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (k, ratio)
    print("inv_s %g sign %+g: worst err / (EPS A) = %.3e" % (inv_s, sign, worst))
