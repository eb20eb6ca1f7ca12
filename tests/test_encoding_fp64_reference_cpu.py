"""The fp64 reference of the permutohedral encoding kernels (oracle/encoding_fp64.py) checked on the CPU at every (D, F):
  * its explicit formulas against fp64 autograd of the straight-through formulation (values from the fp32 weights, their exact
    derivative), for the positions gradient, both lattice gradients and grad_grad_out;
  * its positions gradient against central finite differences of the fp64 encoding at points well inside a simplex;
  * its error model: fp32 arithmetic (the fp32 oracle, oracle/encoding_oracle.py, and its autograd) stays within EPS A / 4 at every
    element of every output, while a table rounded to bf16 or a dropped smallest-weight vertex breaks EPS A. The EPS derivation is in
    the reference's docstring; tests/test_encoding_fp64_gpu.py holds the kernels to EPS A."""
import numpy as np
import pytest
import torch

from oracle import encoding_fp64 as X
from oracle import encoding_oracle as eo

PAIRS = [(D, F) for D in range(2, 7) for F in (1, 2, 4, 8)]


def setup(D, F, N=300, L=5, T=4099, concat=True, seed=0, t=0.55, shift_scale=10.0, sigma_min=1e-3):
    g = torch.Generator().manual_seed(seed * 100 + D * 10 + F)
    pos = torch.rand(N, D, generator=g) - 0.5
    lat = (torch.rand(L, T, F, generator=g) * 2 - 1) * 0.5
    scale = eo.scale_factor([float(s) for s in np.geomspace(1.0, sigma_min, num=L)], D)
    shift = torch.randn(L, D, generator=g) * shift_scale
    window = eo.coarse2fine(L, t) if t is not None else None
    g_out = torch.randn(N, L * F + X.n_extra(D, F, concat), generator=g)
    gg = torch.randn(N, D, generator=g)
    return pos, lat, scale, shift, window, g_out, gg


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


@pytest.mark.parametrize("D,F", PAIRS)
def test_explicit_formulas_match_straight_through_autograd(D, F):
    concat = (D + F) % 2 == 1 or F == 2
    pos, lat, scale, shift, window, g_out, gg = setup(D, F, concat=concat)
    plan = X.plan_of(pos, scale, shift, lat.shape[1])
    pre = torch.randn(lat.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    ref = X.reference(plan, lat, window, concat, 0.5, g_out, gg, pos, prefill=pre, prefill2=2 * pre)
    p = pos.double().requires_grad_(True)
    L64 = lat.double().requires_grad_(True)
    go = g_out.double().requires_grad_(True)
    feat = X.encode_st(p, L64, plan, window, F, concat, 0.5)
    assert rel(ref["out"], feat.detach()) < 1e-12
    gl, gp = torch.autograd.grad(feat, (L64, p), go, create_graph=True)
    dl, dgo = torch.autograd.grad((gp * gg.double()).sum(), (L64, go))
    assert rel(ref["pos_grad"], gp.detach()) < 1e-12
    assert rel(ref["lat"] - pre, gl) < 1e-12
    assert rel(ref["ggo"], dgo) < 1e-12
    assert rel(ref["dlat"] - 2 * pre, dl) < 1e-12
    # the error scales bound their values and vanish only with them
    for k, a in (("out", "A_out"), ("pos_grad", "A_pos"), ("ggo", "A_ggo")):
        assert bool((ref[k].abs() <= ref[a] * (1 + 1e-12)).all()), k
    assert bool(((ref["lat"] - pre).abs() <= ref["lat_A"] * (1 + 1e-12) + 1e-15 * pre.abs()).all())
    assert bool(((ref["dlat"] - 2 * pre).abs() <= ref["dlat_A"] * (1 + 1e-12) + 1e-15 * pre.abs()).all())


@pytest.mark.parametrize("D,F", [(2, 1), (3, 2), (4, 4), (5, 2), (6, 8)])
def test_positions_gradient_matches_finite_differences(D, F):
    """the fp64 encoding (oracle decisions and weights recomputed in fp64 at x +- h) at points whose weights are all >= 0.02"""
    pos, lat, scale, shift, window, g_out, gg = setup(D, F, N=400, L=4, sigma_min=0.1, seed=3)
    keep = torch.ones(pos.shape[0], dtype=torch.bool)
    for l in range(4):
        _, _, b = eo.simplex(pos.double(), scale[l].double(), shift[l].double())
        keep &= (b.min(1).values > 0.02)
    pos, g_out = pos[keep][:50], g_out[keep][:50]
    assert pos.shape[0] >= 10
    plan = X.plan_of(pos, scale, shift, lat.shape[1])
    ref = X.reference(plan, lat, window, True, 0.5, g_out, None, pos)
    h = 1e-6
    lat64, win64 = lat.double(), window.double()
    fd = torch.zeros(pos.shape[0], D, dtype=torch.float64)
    for j in range(D):
        e = torch.zeros(D, dtype=torch.float64)
        e[j] = h
        f = lambda x: (eo.encode(x, lat64, scale.double(), shift.double(), win64, True, 0.5) * g_out.double()).sum(1)
        fd[:, j] = (f(pos.double() + e) - f(pos.double() - e)) / (2 * h)
    # the oracle's fp64 weights use the fp32 1 / (D + 1), a relative 3e-8 from the exact derivative
    assert rel(fd, ref["pos_grad"]) < 1e-6


# ------------------------------------------------------------------------------------------------ the error model
def fp32_outputs(pos, lat, scale, shift, window, concat, scaling, g_out, gg):
    """the fp32 oracle and its autograd: out, positions gradient, lattice gradient, grad_grad_out, double-backward lattice gradient"""
    p = pos.clone().requires_grad_(True)
    lt = lat.clone().requires_grad_(True)
    go = g_out.clone().requires_grad_(True)
    out = eo.encode(p, lt, scale, shift, window, concat, scaling)
    gl, gp = torch.autograd.grad(out, (lt, p), go, create_graph=True)
    dl, dgo = torch.autograd.grad((gp * gg).sum(), (lt, go))
    return dict(out=out.detach(), pos_grad=gp.detach(), lat=gl.detach(), ggo=dgo.detach(), dlat=dl.detach())


def ratios(got, ref):
    """worst err / (EPS A) of every output (the lattice gradients against their per-entry bounds)"""
    r = {}
    for k, a, eps in (("out", "A_out", X.EPS_FWD), ("pos_grad", "A_pos", X.EPS_POS), ("ggo", "A_ggo", X.EPS_GGO)):
        r[k] = X.worst((got[k].double() - ref[k]).abs(), eps * ref[a])
    r["lat"] = X.worst((got["lat"].double() - ref["lat"]).abs(), X.lattice_bound(ref["lat"], ref["lat_A"], ref["lat_n"], None, X.M_LAT))
    r["dlat"] = X.worst((got["dlat"].double() - ref["dlat"]).abs(),
                        X.lattice_bound(ref["dlat"], ref["dlat_A"], ref["dlat_n"], None, X.M_DLAT))
    return r


ERR_CASES = [dict(L=5, t=0.55), dict(L=7, t=None, concat=False), dict(L=32, t=0.8, sigma_min=1e-4)]


@pytest.mark.parametrize("case", range(len(ERR_CASES)))
@pytest.mark.parametrize("D,F", PAIRS)
def test_fp32_arithmetic_within_quarter_eps(D, F, case):
    kw = dict(ERR_CASES[case])
    concat = kw.pop("concat", True)
    pos, lat, scale, shift, window, g_out, gg = setup(D, F, N=200, T=4099, concat=concat, seed=case, **kw)
    plan = X.plan_of(pos, scale, shift, lat.shape[1])
    ref = X.reference(plan, lat, window, concat, 0.5, g_out, gg, pos)
    r = ratios(fp32_outputs(pos, lat, scale, shift, window, concat, 0.5, g_out, gg), ref)
    print("D=%d F=%d case %d fp32: " % (D, F, case) + " ".join("%s %.3f" % kv for kv in r.items()))
    for k in ("out", "pos_grad", "ggo"):
        assert r[k] <= 0.25, (k, r[k])
    # the lattice bounds count every rounding at its worst (<= u each), with no factor to spare when an entry has one contribution
    for k in ("lat", "dlat"):
        assert r[k] <= 1.0, (k, r[k])


def _dropped_simplex(simplex):
    def fn(pos, scale_l, shift_l):
        rem0, rank, bary = simplex(pos, scale_l, shift_l)
        keep = torch.ones_like(bary)
        keep.scatter_(1, bary.detach().abs().argmin(1, keepdim=True), 0.0)
        return rem0, rank, bary * keep
    return fn


@pytest.mark.parametrize("D,F", [(2, 1), (3, 2), (4, 8), (5, 4), (6, 2)])
def test_perturbed_arithmetic_breaks_eps(D, F, monkeypatch):
    """a bf16 table breaks every output that reads the table (the lattice gradients do not); a dropped smallest-weight vertex breaks
    every output"""
    pos, lat, scale, shift, window, g_out, gg = setup(D, F, N=200, L=7, concat=True, seed=9)
    plan = X.plan_of(pos, scale, shift, lat.shape[1])
    ref = X.reference(plan, lat, window, True, 0.5, g_out, gg, pos)
    r = ratios(fp32_outputs(pos, lat.bfloat16().float(), scale, shift, window, True, 0.5, g_out, gg), ref)
    print("D=%d F=%d bf16 table: " % (D, F) + " ".join("%s %.3g" % kv for kv in r.items()))
    for k in ("out", "pos_grad", "ggo"):
        assert r[k] > 1.0, (k, r[k])
    monkeypatch.setattr(eo, "simplex", _dropped_simplex(eo.simplex))
    r = ratios(fp32_outputs(pos, lat, scale, shift, window, True, 0.5, g_out, gg), ref)
    print("D=%d F=%d dropped vertex: " % (D, F) + " ".join("%s %.3g" % kv for kv in r.items()))
    for k, v in r.items():
        assert v > 1.0, (k, v)


def test_gpu_cases_cover_the_edges():
    """every value the GPU test promises appears somewhere in its parametrisation"""
    import test_encoding_fp64_gpu as G
    cases = [G.CASES[i] for i in range(len(G.CASES))]
    assert sorted({c.D for c in cases}) == [2, 3, 4, 5, 6] and {(c.D, c.F) for c in cases} == set(PAIRS)
    Ns = {c.N for c in cases}
    assert {1, 31, 32, 33, 4097} <= Ns and max(Ns) >= 40000
    assert {1, 5, 7, 32} <= {c.L for c in cases}
    assert {1, 3, 4099, 2 ** 14, 2 ** 20 + 7} <= {c.T for c in cases}
    assert {False, True} <= {c.concat for c in cases}
    assert any(c.concat and (c.D + c.F - 1) // c.F > 1 for c in cases), "concat with more than one group"
    assert any(c.concat and c.D % c.F for c in cases), "concat with pad columns"
    assert {"none", "open", "partial", "closed"} <= {c.window for c in cases}
    assert {"uniform", "clustered", "lattice", "negative", "large"} <= {c.layout for c in cases}
