"""The fp64 forward references (oracle/backward_fp64.py: sdf_forward_reference, rgb_forward_reference, bg_forward_reference) checked on
the CPU: their values against the original project's own Python (tests/golden/refpy_golden*.npz), their tangent streams against fp64
autograd, and their error scales A against an emulation of the kernels' arithmetic.

The tolerance of the GPU test (tests/test_fused_forward_fp64_gpu.py) is |got - ref| <= EPS A per element. EPS comes from the error
analysis of the kernels' products: an operand split x = hi + lo into two bf16 leaves |x - hi - lo| <= 2^-17 |x| (2^-16 at worst), a
product hi hi + hi lo + lo hi drops lo lo (2^-16 of the term) and accumulates in fp32, so one layer adds ~3 2^-17 of its terms' scale
A (their quadrature sum, see oracle/backward_fp64.py); four SDF layers give 12 2^-17 = 2^-13.4, the seven background layers 21 2^-17 =
2^-12.6. EPS = 2^-12 covers both; the north star's 1e-3 is the ceiling it must never be raised past. The emulation below (bf16 hi / lo
splits of operands and weights, the three products, fp32 accumulation, the kernels' fp32 GELU) stays below EPS A / 4 at every element
of the GPU cases' shapes (observed: below 2^-15.5 A), and a one-pass bf16 product (hi hi only, error 2^-9 of a term) breaks the bound
(observed: above 2^-9 A): that is the sensitivity the GPU test has."""
import numpy as np
import pytest
import torch

from oracle import backward_fp64 as R
from test_backward_fp64_reference_cpu import G, _lattice_from_seed, _t, rel  # noqa: F401  (G: the fixtures)
from test_fused_forward_fp64_gpu import BG_LEVELS, EPS, RGB_HIDDEN, RGB_LEVELS, SDF_SHAPES


# ------------------------------------------------------------------------------------------------ the original project's fixtures
def test_sdf_forward_reference_matches_original_python(G):
    L, T = 24, 2 ** 18
    W = [_t(G["sdf.mlp_sdf.%d.weight" % i]) for i in (0, 2, 4, 6)]
    b = [_t(G["sdf.mlp_sdf.%d.bias" % i]) for i in (0, 2, 4, 6)]
    win = R.window_of(L, 0.3 + 0.7 * int(G["sdf_in.iter"]) / 10000)
    ref = R.sdf_forward_reference(_t(G["sdf_in.points"]), _lattice_from_seed(11, L, T, 2, 0.3), R.level_scales(L, 3),
                                  _t(G["sdf.encoding.random_shift_per_level"]), win, 1e-3, W, b)
    assert rel(ref["sdf"], G["sdf_out.sdf"]) < 1e-4
    assert rel(ref["grad"], G["sdf_out.grad"]) < 1e-4
    assert rel(ref["geom"], G["sdf_out.geom"]) < 1e-4


def test_rgb_forward_reference_matches_original_python(G):
    """colour head (calibration, sigmoid) applied in fp64 around the linear output, the matrices normalised in fp64 from the raw
    weights and bounds"""
    L, T = 24, 2 ** 18
    W_eff = [R.lipschitz_weights(_t(G["rgb.mlp.layers.%d.weight" % i]), _t(G["rgb.mlp.lipshitz_bound_per_layer.%d" % i])) for i in range(4)]
    b = [_t(G["rgb.mlp.layers.%d.bias" % i]) for i in range(4)]
    pts, dirs, sg, gm = (_t(G["rgb_in." + k]) for k in ("points", "dirs", "sdf_gradients", "geom"))
    x = R.rgb_forward_reference(pts, dirs, sg, gm, _lattice_from_seed(12, L, T, 2, 0.3), R.level_scales(L, 3),
                                _t(G["rgb.encoding.random_shift_per_level"]), R.window_of(L, 1.0), 1.0, W_eff, b)["out"]
    se = G["rgb_in.ray_start_end_idx"]
    img = _t(G["rgb_in.img_indices"]).long()[torch.from_numpy(np.repeat(np.arange(se.shape[0]), se[:, 1] - se[:, 0]))]
    wd, bs = _t(G["cal.weight_delta"]).double()[img], _t(G["cal.bias"]).double()[img]
    fixed = (img == 0)[:, None]
    wd, bs = torch.where(fixed, torch.zeros_like(wd), wd), torch.where(fixed, torch.zeros_like(bs), bs)
    assert rel(torch.sigmoid(x * (1 + wd) + bs), G["rgb_out.rgb"]) < 1e-4


def test_background_forward_reference_matches_original_python(G):
    L, T = 24, 2 ** 18
    keys = ["bg.mlp_feat_and_density.%d" % i for i in (0, 2, 4, 6)] + ["bg.mlp_rgb.%d" % i for i in (0, 2, 4)]
    W, b = [_t(G[k + ".weight"]) for k in keys], [_t(G[k + ".bias"]) for k in keys]
    ref = R.bg_forward_reference(_t(G["bg_in.points"]), _t(G["bg_in.dirs"]), _lattice_from_seed(13, L, T, 2, 0.3), R.level_scales(L, 4),
                                 _t(G["bg.encoding.random_shift_per_level"]), R.window_of(L, 1.0), 1.0, W, b)
    assert rel(torch.sigmoid(ref["rgb_raw"]), G["bg_out.rgb"]) < 1e-4
    assert rel(ref["density"], G["bg_out.density"]) < 1e-4


# ------------------------------------------------------------------------------------------------ tangents
def sdf_case(L, hidden, out_dim, N, T=5003, seed=0, layout="uniform", win_t=0.6):
    g = torch.Generator().manual_seed(seed)
    if layout == "ray":            # 64 samples 1/128 of the bounding sphere's diameter apart along random rays
        nr = (N + 63) // 64
        o = (torch.rand(nr, 3, generator=g) - 0.5) * 0.5
        d = torch.nn.functional.normalize(torch.randn(nr, 3, generator=g), dim=1)
        pos = (o[:, None, :] + (torch.arange(64.0) / 128)[None, :, None] * d[:, None, :]).reshape(-1, 3)[:N].contiguous()
    else:
        pos = (torch.rand(N, 3, generator=g) - 0.5) * 0.9
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    dims = [2 * L + 4, hidden, hidden, hidden, out_dim]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    return pos, lat, R.level_scales(L, 3), shift, R.window_of(L, win_t), W, b


@pytest.mark.parametrize("shape", [(8, 32, 9), (4, 16, 1), (28, 48, 33)])
def test_sdf_forward_tangents_match_autograd(shape):
    """grad = the three tangent streams of the forward, against fp64 autograd through encode_st + the MLP wrt the position"""
    L, hidden, out_dim = shape
    pos, lat, scale, shift, win, W, b = sdf_case(L, hidden, out_dim, 300, seed=L)
    ref = R.sdf_forward_reference(pos, lat, scale, shift, win, 1e-3, W, b)
    plan = R.Plan(pos, scale, shift, lat.shape[1])
    p = pos.double().requires_grad_(True)
    h = R.encode_st(p, lat.double(), plan, win, 1e-3)
    for l in range(4):
        h = torch.nn.functional.linear(h, W[l].double(), b[l].double())
        if l < 3:
            h = torch.nn.functional.gelu(h)
    gx = torch.autograd.grad(h[:, 0].sum(), p)[0]
    assert rel(ref["grad"], gx) < 1e-12
    assert rel(ref["sdf"], h[:, 0].detach()) < 1e-12
    assert out_dim == 1 or rel(ref["geom"], h[:, 1:].detach()) < 1e-12
    for k in ("sdf", "grad", "geom"):
        assert bool(torch.isfinite(ref["A_" + k]).all() and (ref["A_" + k] > 0).all()), k


# ------------------------------------------------------------------------------------------------ the error model
def _split(x):
    hi = x.to(torch.bfloat16).float()
    return hi, (x - hi).to(torch.bfloat16).float()


class Emulated(R.Exact):
    """the kernels' arithmetic: bf16 hi / lo splits of the operand and the weights, the products `products` ("hh", "hl", "lh": the
    kernels form all three) summed in fp32, the bias added in fp32, and the kernels' fp32 GELU (gelu_eval of fused_common.cuh:
    Abramowitz-Stegun 7.1.26 for Phi)"""

    def __init__(self, products=("hh", "hl", "lh")):
        self.products = products

    def linear(self, l, a, W, b=None):
        (ah, al), (wh, wl) = _split(a.float()), _split(W.float())
        terms = {"hh": (ah, wh), "hl": (ah, wl), "lh": (al, wh)}
        z = None
        for p in self.products:
            x, w = terms[p]
            z = x @ w.t() if z is None else z + x @ w.t()
        return z + b.float() if b is not None else z

    def gelu(self, z):
        z = z.float()
        E = torch.exp(-0.5 * z * z)
        t = 1.0 / (0.3275911 * 0.70710678118654752 * z.abs() + 1.0)
        poly = t * (0.254829592 + t * (-0.284496736 + t * (1.421413741 + t * (-1.453152027 + t * 1.061405429))))
        q = 0.5 * poly * E
        cdf = torch.where(z >= 0, 1.0 - q, q)
        return z * cdf, z * (0.3989422804014327 * E) + cdf


def ratio(got, ref, A):
    return float(((got.double() - ref.double()).abs() / (EPS * A)).max())


def sdf_ratios(ar, shape, N=2048, seed=0, layout="uniform"):
    L, hidden, out_dim = shape
    pos, lat, scale, shift, win, W, b = sdf_case(L, hidden, out_dim, N, seed=seed, layout=layout)
    plan = R.Plan(pos, scale, shift, lat.shape[1])
    ref = R.sdf_forward_reference(pos, lat, scale, shift, win, 1e-3, W, b, plan=plan)
    emu = R.sdf_forward_reference(pos, lat, scale, shift, win, 1e-3, W, b, plan=plan, arith=ar)
    return {k: ratio(emu[k], ref[k], ref["A_" + k]) for k in ("sdf", "grad", "geom") if ref[k].numel()}


def rgb_ratios(ar, L, hs, N=2048, seed=0):
    g = torch.Generator().manual_seed(seed)
    pos = (torch.rand(N, 3, generator=g) - 0.5) * 0.8
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1)
    sg, gm = torch.randn(N, 3, generator=g) * 2, torch.randn(N, 32, generator=g)
    lat = (torch.rand(L, 5003, 2, generator=g) * 2 - 1) * 0.3
    dims = [2 * L + 64] + list(hs) + [3]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    args = (pos, dirs, sg, gm, lat, R.level_scales(L, 3), torch.randn(L, 3, generator=g) * 10, R.window_of(L, 0.6), 1.0, W, b)
    sh = R.sh_fp32(dirs, 5)
    ref = R.rgb_forward_reference(*args, sh=sh)
    emu = R.rgb_forward_reference(*args, sh=sh, arith=ar)
    return {"out": ratio(emu["out"], ref["out"], ref["A_out"])}


def bg_ratios(ar, L, N=2048, seed=0):
    g = torch.Generator().manual_seed(seed)
    pos = torch.cat([torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1), torch.rand(N, 1, generator=g)], 1)
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1)
    lat = (torch.rand(L, 5003, 2, generator=g) * 2 - 1) * 0.3
    dims = [(2 * L + 4, 64), (64, 64), (64, 64), (64, 65), (80, 64), (64, 64), (64, 3)]
    W = [torch.randn(o, i, generator=g) / i ** 0.5 for i, o in dims]
    b = [torch.randn(o, generator=g) * 0.1 for _, o in dims]
    W[3][0] *= 20.0                 # a density pre-activation far from 0 on both sides
    args = (pos, dirs, lat, R.level_scales(L, 4), torch.randn(L, 4, generator=g) * 10, R.window_of(L, 0.6), 1.0, W, b)
    sh = R.sh_fp32(dirs, 4)
    ref = R.bg_forward_reference(*args, sh=sh)
    emu = R.bg_forward_reference(*args, sh=sh, arith=ar)
    return {"rgb_raw": ratio(emu["rgb_raw"], ref["rgb_raw"], ref["A_rgb"]),
            "density": ratio(emu["density"], ref["density"], ref["A_density"])}


def test_eps_within_the_north_star():
    assert EPS <= 2.0 ** -12 and EPS < 1e-3


@pytest.mark.parametrize("shape", SDF_SHAPES, ids=["L%d-h%d-o%d" % s for s in SDF_SHAPES])
def test_sdf_error_model_holds_for_the_kernel_arithmetic(shape):
    """the emulated kernel arithmetic stays within EPS A / 4 at every element; a one-pass bf16 product does not stay within EPS A"""
    for layout in ("uniform", "ray"):
        r = sdf_ratios(Emulated(), shape, layout=layout, seed=sum(shape))
        print("sdf", shape, layout, r)
        assert max(r.values()) <= 0.25, (shape, layout, r)
    one = sdf_ratios(Emulated(("hh",)), shape, seed=sum(shape))
    print("sdf one-pass", shape, one)
    assert one["sdf"] > 1.0 and one["grad"] > 1.0, (shape, one)


@pytest.mark.parametrize("hs", RGB_HIDDEN, ids=["h%d.%d.%d" % h for h in RGB_HIDDEN])
def test_rgb_error_model_holds_for_the_kernel_arithmetic(hs):
    for L in RGB_LEVELS:
        r = rgb_ratios(Emulated(), L, hs, seed=L)
        print("rgb", L, hs, r)
        assert r["out"] <= 0.25, (L, hs, r)
    one = rgb_ratios(Emulated(("hh",)), 16, hs, N=4096)
    print("rgb one-pass", hs, one)
    assert one["out"] > 1.0, (hs, one)


def test_background_error_model_holds_for_the_kernel_arithmetic():
    for L in BG_LEVELS:
        r = bg_ratios(Emulated(), L, seed=L)
        print("bg", L, r)
        assert max(r.values()) <= 0.25, (L, r)
    one = bg_ratios(Emulated(("hh",)), 16, N=4096)
    print("bg one-pass", one)
    assert one["rgb_raw"] > 1.0 and one["density"] > 1.0, one
