"""CPU checks of the fp64 ray-path reference (oracle/raypath_fp64.py): the serial fp32 C oracle (oracle/rayops_oracle.c), which the
GPU kernels match bit for bit (or within __expf for the NeRF render), must sit inside the reference's error bound on the layouts the
GPU tests use -- ragged rays with gaps and skipped rays, and the equal layout. A wrong derivative in the oracle, or a bound too tight
for a correct fp32 chain, fails here without a GPU."""
import numpy as np
import pytest

from oracle import rayops as orc
from oracle import raypath_fp64 as rf


def _packed(se, M, equal=False, fixed_n=0):
    R = se.shape[0]
    p = orc.Packed(R, M)
    p.start_end, p.max_nr_samples, p.equal, p.fixed_n = orc.i32(se), M, equal, fixed_n
    return p


def _layouts():
    se, M = rf.ragged_layout(seed=1)
    yield "ragged", se, M, False, 0
    for fixed_n in (1, 16, 32, 33):
        R = 37
        yield "equal%d" % fixed_n, np.zeros((R, 2), np.int32), R * fixed_n - fixed_n, True, fixed_n    # the last ray is skipped


LAYOUTS = list(_layouts())


@pytest.mark.parametrize("case", LAYOUTS, ids=[c[0] for c in LAYOUTS])
def test_oracle_within_fp64_bounds(case):
    name, se, M, equal, fixed_n = case
    R = se.shape[0]
    rng = np.random.RandomState(7)
    p = _packed(se, M, equal, fixed_n)
    lay = rf.layout(se, R, M, equal, fixed_n)
    rep = {}
    # transmittance: factors in (0.5, 1], a few rays with a factor at or below 1e-6
    a = (0.5 + 0.5 * rng.rand(M, 1)).astype(np.float32)
    a[rng.rand(M) < 0.002] = 1e-7
    T, bg = orc.vr_cumprod(p, a)
    ref = rf.cumprod(lay, a)
    rf.check("T", T[:, 0], ref["T"], ref["A_T"], ref["rows"], rep)
    rf.check("bg_T", bg[:, 0], ref["bg"], ref["A_bg"], report=rep)
    gT, gbg = rng.rand(M, 1).astype(np.float32), rng.rand(R, 1).astype(np.float32)
    cs = orc.vr_cumsum(p, (gT * T).astype(np.float32), True)
    ga = orc.vr_cumprod_backward(p, gbg, a, bg, cs)
    ref = rf.cumprod_backward(lay, a, gT, gbg)
    rf.check("cumprod backward", ga[:, 0], ref["g_alpha"], ref["A"], ref["rows"] & rf.rows_of(lay, M, ref["exact_rays"]), rep)
    # integrate and its backward
    w, vals = rng.rand(M, 1).astype(np.float32), (rng.rand(M, 3) - 0.5).astype(np.float32)
    out = orc.vr_integrate(p, vals, w)
    ref = rf.integrate(lay, vals, w)
    rf.check("integrate", out, ref["out"], ref["A"], report=rep)
    gp = (rng.rand(R, 3) - 0.5).astype(np.float32)
    gv, gw = orc.vr_integrate_backward(p, gp, vals, w, False)
    ref = rf.integrate_backward(lay, gp, vals, w)
    rf.check("integrate backward vals", gv, ref["g_vals"], ref["A_vals"], ref["rows"], rep)
    rf.check("integrate backward w", gw[:, 0], ref["g_w"], ref["A_w"], ref["rows"], rep)
    # sums
    for D in (1, 3, 32):
        v = (rng.rand(M, D) - 0.25).astype(np.float32)
        sr, ss = orc.vr_sum(p, v)
        ref = rf.sum_over_each_ray(lay, v)
        rf.check("sum ray D=%d" % D, sr, ref["sum_ray"], ref["A_ray"], report=rep)
        rf.check("sum sample D=%d" % D, ss, ref["sum_sample"], ref["A_sample"], ref["rows"], rep)
        gr, gs = rng.rand(R, D).astype(np.float32), rng.rand(M, D).astype(np.float32)
        ref = rf.sum_over_each_ray_backward(lay, gr, gs)
        rf.check("sum backward D=%d" % D, orc.vr_sum_backward(p, gr, gs), ref["g_vals"], ref["A"], ref["rows"], rep)
    # NeRF render: per-ray density scales put the early-out anywhere along the rays, or nowhere
    rgb = rng.rand(M, 3).astype(np.float32)
    scale = np.exp(rng.uniform(np.log(0.05), np.log(2000.0), R)).astype(np.float32)
    rad = (rng.rand(M, 1) * scale[np.maximum(rf.ray_of_row(lay, M), 0)][:, None]).astype(np.float32)
    p.z = np.cumsum(rng.rand(M, 1) * 0.01, 0).astype(np.float32)
    p.dt = (rng.rand(M, 1) * 0.01).astype(np.float32)
    pr, dp, bgn, wn = orc.vr_render_nerf(p, rgb, rad)
    gp, gb = (rng.rand(R, 3) - 0.5).astype(np.float32), (rng.rand(R, 1) - 0.5).astype(np.float32)
    grgb, grad = orc.vr_render_nerf_backward(p, gp, gb, pr, bgn, rgb, rad)
    ref = rf.volume_render_nerf(lay, rgb, rad, p.z, p.dt, gp, gb)
    ok = ~ref["ambiguous"]
    ok_rows = ref["written"] & rf.rows_of(lay, M, ok)
    rf.check("nerf rgb", pr, ref["pred"], ref["A_pred"], ok, rep)
    rf.check("nerf depth", dp[:, 0], ref["depth"], ref["A_depth"], ok, rep)
    rf.check("nerf bg_T", bgn[:, 0], ref["bg"], ref["A_bg"], ok, rep)
    rf.check("nerf w", wn[:, 0], ref["w"], ref["A_w"], ok_rows, rep)
    rf.check("nerf g_rgb", grgb, ref["g_rgb"], ref["A_g_rgb"], ok_rows, rep)
    rf.check("nerf g_radiance", grad[:, 0], ref["g_rad"], ref["A_g_rad"], ok_rows, rep)
    print("\n%s worst err/bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in sorted(rep.items()))))


def test_nerf_stops_inside_rays():
    """the NeRF layout above exercises the early-out: rays stopped at their first sample, mid-ray, and not at all"""
    se, M = rf.ragged_layout(seed=1)
    R = se.shape[0]
    lay = rf.layout(se, R, M)
    rng = np.random.RandomState(3)
    rad = (rng.rand(M, 1) * 400).astype(np.float32)
    dt = np.full((M, 1), 0.01, np.float32)
    ref = rf.volume_render_nerf(lay, np.zeros((M, 3), np.float32), rad, np.zeros((M, 1), np.float32), dt)
    used = ref["written"].numpy()
    rows = rf.ray_of_row(lay, M)
    per_ray = np.bincount(rows[used & (rows >= 0)], minlength=R)
    n = se[:, 1] - se[:, 0]
    computed = ~lay.skip.numpy() & (n > 0)
    assert (per_ray[computed] < n[computed]).any() and (per_ray[computed] == n[computed]).any()


def test_bounds_catch_a_wrong_derivative():
    """an integrate backward that drops the blue channel (the reference kernel's green-for-blue read) is outside the bound"""
    se, M = rf.ragged_layout(seed=2)
    R = se.shape[0]
    p = _packed(se, M)
    lay = rf.layout(se, R, M)
    rng = np.random.RandomState(0)
    w, vals, gp = rng.rand(M, 1).astype(np.float32), rng.rand(M, 3).astype(np.float32), rng.rand(R, 3).astype(np.float32)
    _, gw = orc.vr_integrate_backward(p, gp, vals, w, True)
    ref = rf.integrate_backward(lay, gp, vals, w)
    with pytest.raises(AssertionError):
        rf.check("integrate backward w (reference bug)", gw[:, 0], ref["g_w"], ref["A_w"], ref["rows"])
