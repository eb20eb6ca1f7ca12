"""The fp64 reference of the fused backwards (oracle/backward_fp64.py) checked on the CPU: its explicit formulation (tangent stream,
per-sample encoder gradients, index_add lattice scatter) against fp64 autograd through the whole forward, central finite differences,
and the fixtures produced by the original project's own Python (tests/golden/refpy_golden*.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import backward_fp64 as R

HERE = os.path.dirname(os.path.abspath(__file__))


def rel(a, b):
    a, b = torch.as_tensor(a).double().reshape(-1), torch.as_tensor(b).double().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


def _sdf_case(N=300, L=8, T=2 ** 10, hidden=32, out_dim=9, seed=0):
    g = torch.Generator().manual_seed(seed)
    pos = (torch.rand(N, 3, generator=g) - 0.5) * 0.9
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    dims = [2 * L + 4, hidden, hidden, hidden, out_dim]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    up = (torch.randn(N, generator=g), torch.randn(N, 3, generator=g), torch.randn(N, out_dim - 1, generator=g))
    return pos, lat, R.level_scales(L, 3), shift, R.window_of(L, 0.6), W, b, up


def test_sdf_explicit_matches_double_backward():
    pos, lat, scale, shift, win, W, b, (gs, gg, gm) = _sdf_case()
    ref = R.sdf_reference(pos, lat, scale, shift, win, 1e-3, W, b, gs, gg, gm)
    lg, gW, gb, _ = R.sdf_autograd(pos, lat, scale, shift, win, 1e-3, W, b, gs, gg, gm)
    assert rel(R.dense_lattice(ref["lattice"]), lg) < 1e-12
    for l in range(4):
        assert rel(ref["W"][l], gW[l]) < 1e-12 and rel(ref["b"][l], gb[l]) < 1e-12, l
    # the window of this ramp position closes the finest levels: their gradient is exactly zero, the partial level's is not
    dense = R.dense_lattice(ref["lattice"])
    w = win.double()
    for l in range(8):
        assert (float(dense[l].abs().max()) == 0.0) == (float(w[l]) == 0.0), l


@pytest.mark.parametrize("which", ["g_sdf", "g_grad", "g_geom"])
def test_sdf_single_upstream_matches_double_backward(which):
    """each upstream alone (the others NULL, as the C ABI allows)"""
    pos, lat, scale, shift, win, W, b, (gs, gg, gm) = _sdf_case(N=200, L=4, T=5003, hidden=16, out_dim=5, seed=1)
    up = {"g_sdf": gs, "g_grad": gg, "g_geom": gm}
    args = [up[k] if k == which else None for k in ("g_sdf", "g_grad", "g_geom")]
    ref = R.sdf_reference(pos, lat, scale, shift, win, 1e-3, W, b, *args)
    lg, gW, gb, _ = R.sdf_autograd(pos, lat, scale, shift, win, 1e-3, W, b, *args)
    assert rel(R.dense_lattice(ref["lattice"]), lg) < 1e-12
    for l in range(4):
        assert rel(ref["W"][l], gW[l]) < 1e-12, l


def test_sdf_finite_differences():
    """central differences in fp64 of the loss (with d sdf / dx from autograd) against the explicit gradients"""
    pos, lat, scale, shift, win, W, b, (gs, gg, gm) = _sdf_case(N=24, L=4, T=64, hidden=16, out_dim=5, seed=2)
    lat, W, b = lat.double(), [w.double() for w in W], [x.double() for x in b]
    ref = R.sdf_reference(pos, lat, scale, shift, win, 1e-3, W, b, gs, gg, gm)
    dense = R.dense_lattice(ref["lattice"])
    loss = lambda lt, Ws, bs: float(R.sdf_autograd(pos, lt, scale, shift, win, 1e-3, Ws, bs, gs, gg, gm)[3])
    h = 1e-5
    nz = torch.nonzero(dense.abs() > 1e-3 * float(dense.abs().max()))
    g = torch.Generator().manual_seed(3)
    for k in torch.randperm(nz.shape[0], generator=g)[:6]:
        i = tuple(nz[k].tolist())
        lp, lm = lat.clone(), lat.clone()
        lp[i] += h
        lm[i] -= h
        fd = (loss(lp, W, b) - loss(lm, W, b)) / (2 * h)
        assert abs(fd - float(dense[i])) < 1e-6 * float(dense.abs().max()), (i, fd, float(dense[i]))
    for l, (r, c) in [(0, (3, 2 * 4 + 1)), (1, (5, 7)), (3, (0, 2)), (3, (2, 11))]:
        Wp, Wm = [w.clone() for w in W], [w.clone() for w in W]
        Wp[l][r, c] += h
        Wm[l][r, c] -= h
        fd = (loss(lat, Wp, b) - loss(lat, Wm, b)) / (2 * h)
        assert abs(fd - float(ref["W"][l][r, c])) < 1e-6 * float(ref["W"][l].abs().max()), (l, r, c)


def test_rgb_and_background_explicit_match_autograd():
    g = torch.Generator().manual_seed(4)
    N, L, T = 257, 8, 5003
    pos = (torch.rand(N, 3, generator=g) - 0.5) * 0.8
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1)
    sg, gm = torch.randn(N, 3, generator=g) * 2, torch.randn(N, 32, generator=g)
    lat = (torch.rand(L, T, 2, generator=g) * 2 - 1) * 0.3
    shift = torch.randn(L, 3, generator=g) * 10
    dims = [2 * L + 64, 64, 48, 32, 3]
    W = [torch.randn(dims[i + 1], dims[i], generator=g) / dims[i] ** 0.5 for i in range(4)]
    b = [torch.randn(dims[i + 1], generator=g) * 0.1 for i in range(4)]
    go = torch.randn(N, 3, generator=g)
    win = R.window_of(L, 0.55)
    ref = R.rgb_reference(pos, dirs, sg, gm, lat, R.level_scales(L, 3), shift, win, 1.0, W, b, go)
    lg, gW, gb, gsg, ggm = R.rgb_autograd(pos, dirs, sg, gm, lat, R.level_scales(L, 3), shift, win, 1.0, W, b, go)
    assert rel(R.dense_lattice(ref["lattice"]), lg) < 1e-12
    assert rel(ref["g_sdf_grad"], gsg) < 1e-12 and rel(ref["g_geom"], ggm) < 1e-12
    for l in range(4):
        assert rel(ref["W"][l], gW[l]) < 1e-12 and rel(ref["b"][l], gb[l]) < 1e-12, l
    # background: 4-D positions, 7 layers
    pos4 = torch.cat([torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1), torch.rand(N, 1, generator=g)], 1)
    dims = [(2 * L + 4, 64), (64, 64), (64, 64), (64, 65), (80, 64), (64, 64), (64, 3)]
    W = [torch.randn(o, i, generator=g) / i ** 0.5 for i, o in dims]
    b = [torch.randn(o, generator=g) * 0.1 for _, o in dims]
    grgb, gden = torch.randn(N, 3, generator=g), torch.randn(N, 1, generator=g)
    shift4 = torch.randn(L, 4, generator=g) * 10
    ref = R.bg_reference(pos4, dirs, lat, R.level_scales(L, 4), shift4, win, 1.0, W, b, grgb, gden)
    lg, gW, gb = R.bg_autograd(pos4, dirs, lat, R.level_scales(L, 4), shift4, win, 1.0, W, b, grgb, gden)
    assert rel(R.dense_lattice(ref["lattice"]), lg) < 1e-12
    for l in range(7):
        assert rel(ref["W"][l], gW[l]) < 1e-12 and rel(ref["b"][l], gb[l]) < 1e-12, l


# ------------------------------------------------------------------------------------------------ the original project's fixtures
@pytest.fixture(scope="module")
def G():
    g = dict(np.load(os.path.join(HERE, "golden", "refpy_golden.npz")))
    g.update(np.load(os.path.join(HERE, "golden", "refpy_golden_bg.npz")))
    return g


def _lattice_from_seed(seed, L, T, F, amp):          # the generator of tests/golden/make_refpy_golden.py
    g = torch.Generator().manual_seed(int(seed))
    return ((torch.rand(L, T, F, generator=g) * 2 - 1) * amp).contiguous()


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def _check_rows(dense, rows, vals, tol=1e-4):
    flat = dense.reshape(-1, 2)
    r = torch.from_numpy(rows.astype(np.int64))
    assert rel(flat[r], _t(vals)) < tol
    mask = torch.ones(flat.shape[0], dtype=torch.bool)
    mask[r] = False
    assert float(flat[mask].abs().max()) == 0.0


def test_sdf_reference_matches_original_python(G):
    L, T = 24, 2 ** 18
    W = [_t(G["sdf.mlp_sdf.%d.weight" % i]) for i in (0, 2, 4, 6)]
    b = [_t(G["sdf.mlp_sdf.%d.bias" % i]) for i in (0, 2, 4, 6)]
    it = int(G["sdf_in.iter"])
    win = R.window_of(L, 0.3 + 0.7 * it / 10000)
    ref = R.sdf_reference(_t(G["sdf_in.points"]), _lattice_from_seed(11, L, T, 2, 0.3), R.level_scales(L, 3),
                          _t(G["sdf.encoding.random_shift_per_level"]), win, 1e-3, W, b, _t(G["sdf_in.ca"]), _t(G["sdf_in.cB"]),
                          _t(G["sdf_in.cC"]))
    assert rel(ref["sdf"], G["sdf_out.sdf"]) < 1e-4 and rel(ref["geom"], G["sdf_out.geom"]) < 1e-4
    for k, i in enumerate((0, 2, 4, 6)):
        assert rel(ref["W"][k], G["sdf_grad.mlp_sdf.%d.weight" % i]) < 1e-4, i
        assert rel(ref["b"][k], G["sdf_grad.mlp_sdf.%d.bias" % i]) < 1e-4, i
    _check_rows(R.dense_lattice(ref["lattice"]), G["sdf_grad.lattice_rows"], G["sdf_grad.lattice_vals"])


def test_rgb_reference_matches_original_python(G):
    """the colour head of the fixture (Lipschitz normalisation, calibration, sigmoid) is applied around the reference in fp64"""
    L, T = 24, 2 ** 18
    Wraw = [_t(G["rgb.mlp.layers.%d.weight" % i]).double().requires_grad_(True) for i in range(4)]
    cs = [_t(G["rgb.mlp.lipshitz_bound_per_layer.%d" % i]).double().requires_grad_(True) for i in range(4)]
    W_eff = [w * torch.clamp(torch.nn.functional.softplus(c) / w.abs().sum(1), max=1.0)[:, None] for w, c in zip(Wraw, cs)]
    b = [_t(G["rgb.mlp.layers.%d.bias" % i]) for i in range(4)]
    pts, dirs, sg, gm = (_t(G["rgb_in." + k]) for k in ("points", "dirs", "sdf_gradients", "geom"))
    args = (pts, dirs, sg, gm, _lattice_from_seed(12, L, T, 2, 0.3), R.level_scales(L, 3), _t(G["rgb.encoding.random_shift_per_level"]),
            R.window_of(L, 1.0), 1.0, [w.detach() for w in W_eff], b)
    x = R.rgb_reference(*args, torch.zeros(pts.shape[0], 3))["out"]
    se = G["rgb_in.ray_start_end_idx"]
    ray = torch.from_numpy(np.repeat(np.arange(se.shape[0]), se[:, 1] - se[:, 0]))
    img = _t(G["rgb_in.img_indices"]).long()[ray]
    wd, bs = _t(G["cal.weight_delta"]).double()[img], _t(G["cal.bias"]).double()[img]
    fixed = (img == 0)[:, None]
    wd, bs = torch.where(fixed, torch.zeros_like(wd), wd), torch.where(fixed, torch.zeros_like(bs), bs)
    rgb = torch.sigmoid(x * (1 + wd) + bs)
    assert rel(rgb, G["rgb_out.rgb"]) < 1e-4
    g_out = _t(G["rgb_in.cw"]).double() * rgb * (1 - rgb) * (1 + wd)
    ref = R.rgb_reference(*args, g_out)
    assert rel(ref["g_sdf_grad"], G["rgb_grad.sdf_gradients"]) < 1e-4 and rel(ref["g_geom"], G["rgb_grad.geom"]) < 1e-4
    gW = torch.autograd.grad(W_eff, Wraw + cs, ref["W"])
    for i in range(4):
        assert rel(gW[i], G["rgb_grad.mlp.layers.%d.weight" % i]) < 1e-4, i
        assert rel(ref["b"][i], G["rgb_grad.mlp.layers.%d.bias" % i]) < 1e-4, i
        want = G["rgb_grad.mlp.lipshitz_bound_per_layer.%d" % i]
        assert abs(float(gW[4 + i]) - float(want[0])) <= 1e-4 * max(abs(float(want[0])), 1e-3), i
    _check_rows(R.dense_lattice(ref["lattice"]), G["rgb_grad.lattice_rows"], G["rgb_grad.lattice_vals"])


def test_background_reference_matches_original_python(G):
    L, T = 24, 2 ** 18
    keys = ["bg.mlp_feat_and_density.%d" % i for i in (0, 2, 4, 6)] + ["bg.mlp_rgb.%d" % i for i in (0, 2, 4)]
    W, b = [_t(G[k + ".weight"]) for k in keys], [_t(G[k + ".bias"]) for k in keys]
    pts, dirs = _t(G["bg_in.points"]), _t(G["bg_in.dirs"])
    args = (pts, dirs, _lattice_from_seed(13, L, T, 2, 0.3), R.level_scales(L, 4), _t(G["bg.encoding.random_shift_per_level"]),
            R.window_of(L, 1.0), 1.0, W, b)
    first = R.bg_reference(*args, torch.zeros(pts.shape[0], 3), torch.zeros(pts.shape[0], 1))
    rgb = torch.sigmoid(first["rgb"])
    assert rel(rgb, G["bg_out.rgb"]) < 1e-4 and rel(first["density"], G["bg_out.density"]) < 1e-4
    ref = R.bg_reference(*args, _t(G["bg_in.cb"]).double() * rgb * (1 - rgb), _t(G["bg_in.cd"]))
    for k, gw, gb in zip(keys, ref["W"], ref["b"]):
        assert rel(gw, G[k.replace("bg.", "bg_grad.") + ".weight"]) < 1e-4, k
        assert rel(gb, G[k.replace("bg.", "bg_grad.") + ".bias"]) < 1e-4, k
    _check_rows(R.dense_lattice(ref["lattice"]), G["bg_grad.lattice_rows"], G["bg_grad.lattice_vals"])


def test_barycentric_position_derivative():
    """the position derivative both formulations share: bary_linear reproduces encoding_oracle's weights (fp64, same simplex), and its
    tangent along v equals central differences of encoding_oracle's fp64 weights along v inside the simplex"""
    from oracle import encoding_oracle as eo
    g = torch.Generator().manual_seed(5)
    L, N = 8, 200
    pos = ((torch.rand(N, 3, generator=g) - 0.5) * 0.9).double()
    v = torch.randn(N, 3, generator=g).double()
    scale, shift = R.level_scales(L, 3).double(), (torch.randn(L, 3, generator=g) * 10).double()
    checked = 0
    for l in range(L):
        rem0, rank, bary = eo.simplex(pos, scale[l], shift[l])
        cf = (pos + shift[l]) * scale[l]
        assert float((R.bary_linear(cf, rank, rem0) - bary).abs().max()) < 1e-9 * float(cf.abs().max() + 1)
        h = 1e-3 / float(scale[l].max())
        rp, kp, bp = eo.simplex(pos + h * v, scale[l], shift[l])
        rm, km, bm = eo.simplex(pos - h * v, scale[l], shift[l])
        same = (rp == rem0).all(1) & (kp == rank).all(1) & (rm == rem0).all(1) & (km == rank).all(1)
        fd = (bp - bm) / (2 * h)
        dB = R.bary_linear(v * scale[l], rank)
        assert float((fd - dB)[same].abs().max()) < 1e-6 * float(dB.abs().max()), l
        checked += int(same.sum())
    assert checked > L * N // 2
