"""CPU tests that pin the C ray-path oracle (oracle/rayops_oracle.c): known-answer vectors, structural
invariants, and -- when tests/golden/ref_*.npz exist -- fixtures produced by the reference's own CUDA
kernels (tests/golden/make_ref_golden.py)."""
import glob
import os

import numpy as np
import pytest

import scenes
from oracle import rayops as orc

V = 64


@pytest.fixture(scope="module")
def scene():
    o, d = scenes.make_rays(128, seed=3)
    values, occ = scenes.analytic_occupancy(V)
    pe, te, px, tx, hit = orc.sphere_ray_intersection(scenes.SPHERE_RADIUS, [0, 0, 0], o, d)
    return dict(o=o, d=d, occ=occ.astype(np.uint8), te=te, tx=tx, hit=hit)


def test_pcg32_canonical_stream():
    # canonical pcg32-demo stream: pcg32_srandom(42, 54) -> state = 0; inc = 54*2+1; step; state += 42; step
    M, inc = 0x5851F42D4C957F2D, (54 << 1) | 1
    state = ((0 * M + inc + 42) * M + inc) & ((1 << 64) - 1)
    u, f = orc.pcg32_draw(6, state=state, inc=inc)
    assert [hex(int(x)) for x in u] == ["0xa15c02b7", "0x7b47f409", "0xba1d3330", "0x83d2f293", "0xbfa4784b", "0xcbed606e"]
    assert np.all((f >= 0) & (f < 1))
    u, f = orc.pcg32_draw(6)        # default state of the reference (pcg32.h:33-34)
    # jump-ahead equals stepping
    u2, _ = orc.pcg32_draw(3, advance=3)
    assert np.array_equal(u2, u[3:6])


def test_morton_roundtrip_all_10bit():
    rng = np.random.RandomState(0)
    xyz = rng.randint(0, 1024, size=(200000, 3)).astype(np.uint32)
    xyz[:4] = [[0, 0, 0], [1023, 1023, 1023], [1, 0, 0], [0, 0, 1]]
    code, back = orc.morton(xyz)
    assert np.array_equal(back, xyz)
    assert code[0] == 0 and code[1] == (1 << 30) - 1 and code[2] == 1 and code[3] == 4


def test_sphere_known_answers():
    o = np.array([[0, 0, -2], [0, 0, -2], [0, 0, 0], [2, 2, 2]], np.float32)
    d = np.array([[0, 0, 1], [0, 1, 0], [1, 0, 0], [0, 0, 1]], np.float32)
    pe, te, px, tx, hit = orc.sphere_ray_intersection(0.5, [0, 0, 0], o, d)
    assert hit[:, 0].tolist() == [True, False, True, False]
    assert te[0, 0] == 1.5 and tx[0, 0] == 2.5
    assert te[1, 0] == 0 and tx[1, 0] == 0 and np.array_equal(pe[1], o[1])          # miss -> origin, t=0
    assert te[2, 0] == 0 and tx[2, 0] == 0.5                                           # inside: entry clamped to 0


def test_sh_degree1_and_orthonormality():
    assert abs(orc.spherical_harmonics(np.array([[0, 0, 1.0]], np.float32), 1)[0, 0] - 0.28209479177387814) < 1e-7
    rng = np.random.RandomState(0)
    d = rng.randn(200000, 3)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    Y = orc.spherical_harmonics(d.astype(np.float32), 7).astype(np.float64)
    G = 4 * np.pi * (Y.T @ Y) / d.shape[0]
    assert np.abs(G - np.eye(49)).max() < 0.05          # Monte-Carlo orthonormality of the real SH basis


def test_occupancy_scene(scene):
    occ = scene["occ"]
    frac = occ.mean()
    assert 0.02 < frac < 0.5, "analytic sphere shell should occupy a thin band"
    pts = np.array([[0.3, 0, 0], [0, 0, 0], [0.49, 0.49, 0.49], [2, 0, 0], [-0.3, 0.0, 0.0]], np.float32)
    got = orc.occ_check_occupancy(V, 1.0, [0, 0, 0], occ, pts)[:, 0].tolist()
    assert got == [True, False, False, False, True]
    # grid centres: morton order, centred grid
    c = orc.occ_grid_points(V, 1.0, [0, 0, 0])
    assert np.allclose(c[0], -0.5 + 0.5 / V) and np.allclose(c[1], [-0.5 + 1.5 / V, -0.5 + 0.5 / V, -0.5 + 0.5 / V])
    assert np.all(orc.occ_check_occupancy(V, 1.0, [0, 0, 0], np.ones(V ** 3, np.uint8), c))
    j = orc.occ_grid_points(V, 1.0, [0, 0, 0], np.arange(100, dtype=np.int32), True)
    assert np.abs(j - c[:100]).max() <= 0.5 / V + 1e-7 and np.abs(j - c[:100]).max() > 0


@pytest.mark.parametrize("jitter", [False, True])
def test_sampling_invariants(scene, jitter):
    o, d = scene["o"], scene["d"]
    p = orc.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], o, d, scene["te"], scene["tx"], scene["occ"], 2e-3, 48, jitter)
    n = p.start_end[:, 1] - p.start_end[:, 0]
    assert n.max() == 48 and (n[~scene["hit"][:, 0]] == 0).all()
    assert ((n == 0) | (n > 2)).all()
    for r in np.nonzero(n)[0]:
        s, e = p.start_end[r]
        z = p.z[s:e, 0]
        assert np.all(np.diff(z) > 0) and z[0] >= scene["te"][r, 0] and z[-1] <= scene["tx"][r, 0]
        assert np.allclose(p.pos[s:e], o[r] + z[:, None] * d[r], atol=1e-6)
        assert np.all(orc.occ_check_occupancy(V, 1.0, [0, 0, 0], scene["occ"], p.pos[s:e])), "samples must lie in occupied voxels"
        assert np.all(p.dt[s:e - 1, 0] == p.fixed_dt[r, 0]) and 0 <= p.dt[e - 1, 0] <= p.fixed_dt[r, 0]
    q = orc.packed_compact(p)
    assert q.cur == n.sum() and np.array_equal(q.start_end[:, 1] - q.start_end[:, 0], n)
    assert np.array_equal(orc.packed_per_sample_ray_idx(q.start_end, q.cur), np.repeat(np.arange(len(n)), n))
    # empty / ragged input
    e = orc.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], o[:0], d[:0], scene["te"][:0], scene["tx"][:0], scene["occ"], 2e-3, 48, jitter)
    assert e.cur == 0


def test_first_sample_and_advance(scene):
    o, d = scene["o"], scene["d"]
    p = orc.occ_first_sample_start(V, 1.0, [0, 0, 0], o, d, scene["te"], scene["tx"], scene["occ"])
    n = p.start_end[:, 1] - p.start_end[:, 0]
    assert set(np.unique(n)) <= {0, 1} and n.sum() > 50
    sel = np.nonzero(n)[0]
    assert np.all(orc.occ_check_occupancy(V, 1.0, [0, 0, 0], scene["occ"], p.pos[p.start_end[sel, 0]]))
    # axis-aligned rays only creep by eps per step (reference quirk, SURVEY.md A.3): leave them out of the march test
    sel = sel[np.abs(d[sel]).min(1) > 1e-3]
    inside = (0.1 * d[sel]).astype(np.float32)           # points near the centre (empty), marching outwards
    newpos, within = orc.occ_advance_to_next_occupied(V, 1.0, [0, 0, 0], d[sel], inside, scene["occ"])
    assert within.all() and np.all(orc.occ_check_occupancy(V, 1.0, [0, 0, 0], scene["occ"], newpos))
    # leaving through a positive face is detected (index >= V^3); leaving through a negative face is not, because the
    # float->uint cast saturates to voxel 0 (reference quirk, SURVEY.md A.2) -- so march along |d|
    da = np.abs(d[sel])
    out, w2 = orc.occ_advance_to_next_occupied(V, 1.0, [0, 0, 0], da, (0.45 * da).astype(np.float32), scene["occ"])
    assert not w2.any(), "marching outwards from outside the shell leaves the grid"


def test_volume_rendering_against_numpy(scene):
    o, d = scene["o"], scene["d"]
    p = orc.packed_compact(orc.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], o, d, scene["te"], scene["tx"], scene["occ"], 2e-3, 48))
    N = p.cur
    rng = np.random.RandomState(1)
    a = rng.uniform(0.8, 1.0, (N, 1)).astype(np.float32)
    w = rng.rand(N, 1).astype(np.float32)
    rgb = rng.rand(N, 3).astype(np.float32)
    T, bg = orc.vr_cumprod(p, a)
    s_ray, s_smp = orc.vr_sum(p, w)
    integ = orc.vr_integrate(p, rgb, w)
    cdf = orc.vr_cdf(p, w)
    cs_f, cs_r = orc.vr_cumsum(p, w, False), orc.vr_cumsum(p, w, True)
    for r, (s, e) in enumerate(p.start_end):
        if e == s:
            assert bg[r, 0] == 1 and s_ray[r, 0] == 0
            continue
        ref_T = np.concatenate([[1.0], np.cumprod(a[s:e - 1, 0].astype(np.float64))])
        assert np.allclose(T[s:e, 0], ref_T, rtol=1e-5) and np.isclose(bg[r, 0], ref_T[-1], rtol=1e-5)
        assert np.isclose(s_ray[r, 0], w[s:e].sum(), rtol=1e-5) and np.allclose(s_smp[s:e], s_ray[r])
        assert np.allclose(integ[r], (w[s:e] * rgb[s:e]).sum(0), rtol=1e-5)
        assert cdf[s, 0] == 0 and np.allclose(cdf[s:e, 0], np.concatenate([[0], np.cumsum(w[s:e - 1, 0])]), rtol=1e-5)
        assert np.allclose(cs_f[s:e, 0], np.cumsum(w[s:e, 0]), rtol=1e-5) and np.allclose(cs_r[s:e, 0], np.cumsum(w[s:e, 0][::-1])[::-1], rtol=1e-5)
    # sdf2alpha on an analytic sdf, and a full importance-resampling round
    sdf = scenes.analytic_sdf(p.pos)
    alpha = np.clip(orc.vr_sdf2alpha(p, sdf, 512, True, 1.0), 0, 1)
    assert alpha.min() >= 0 and alpha.max() <= 1 and alpha.max() > 0.05
    for s, e in p.start_end:
        if e > s:
            assert alpha[e - 1, 0] == 0
    T2, _ = orc.vr_cumprod(p, 1 - alpha + 1e-7)
    ww = alpha * T2
    _, ws = orc.vr_sum(p, ww)
    ww = ww / np.maximum(ws, 1e-6)
    cdf = orc.vr_cdf(p, ww)
    p.sdf, p.has_sdf = sdf, True
    q = orc.vr_importance_sample(o, d, p, cdf, 16, False)
    q.sdf, q.has_sdf = scenes.analytic_sdf(q.pos), True
    nz = (p.start_end[:, 1] - p.start_end[:, 0]) > 0
    zq = q.z.reshape(-1, 16)
    assert np.all(zq[~nz] == -1) and np.all(np.diff(zq[nz], axis=1) >= -1e-6)
    # importance samples concentrate around the surface |x| = 0.3
    assert np.median(np.abs(np.linalg.norm(q.pos.reshape(-1, 16, 3)[nz], axis=2) - 0.3)) < 0.02
    c = orc.vr_combine(o, d, scene["tx"], p, q)
    n_u = p.start_end[:, 1] - p.start_end[:, 0]
    assert np.array_equal(c.start_end[:, 1] - c.start_end[:, 0], np.where(n_u > 1, n_u + 16, 0))
    for r, (s, e) in enumerate(c.start_end):
        if e > s:
            assert np.all(np.diff(c.z[s:e, 0]) >= 0) and np.all(c.dt[s:e, 0] <= c.fixed_dt[r, 0] + 1e-7)
            assert np.allclose(c.sdf[s:e], scenes.analytic_sdf(c.pos[s:e]), atol=1e-5)


def test_backward_kernels_against_finite_differences(scene):
    o, d = scene["o"], scene["d"]
    p = orc.packed_compact(orc.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], o[:16], d[:16], scene["te"][:16], scene["tx"][:16],
                                                               scene["occ"], 5e-3, 12))
    N, R = p.cur, 16
    rng = np.random.RandomState(2)
    a = rng.uniform(0.5, 1.0, (N, 1)).astype(np.float32)
    gT, gbg = rng.randn(N, 1).astype(np.float32), rng.randn(R, 1).astype(np.float32)
    T, bg = orc.vr_cumprod(p, a)
    cs = orc.vr_cumsum(p, gT * T, True)
    ga = orc.vr_cumprod_backward(p, gbg, a, bg, cs)

    def f(aa):
        T_, bg_ = orc.vr_cumprod(p, aa.astype(np.float32))
        return float((T_.astype(np.float64) * gT).sum() + (bg_.astype(np.float64) * gbg).sum())
    for i in rng.choice(N, 10, replace=False):
        da = np.zeros_like(a); da[i] = 1e-3
        fd = (f(a + da) - f(a - da)) / 2e-3
        assert abs(fd - ga[i, 0]) < 2e-2 * (1 + abs(fd))
    # integrate backward: fixed vs reference-bug mode differ only in the blue term of g_w
    rgb, w, gp = rng.rand(N, 3).astype(np.float32), rng.rand(N, 1).astype(np.float32), rng.randn(R, 3).astype(np.float32)
    gv, gw = orc.vr_integrate_backward(p, gp, rgb, w, False)
    gv2, gw2 = orc.vr_integrate_backward(p, gp, rgb, w, True)
    ridx = orc.packed_per_sample_ray_idx(p.start_end, N)
    assert np.allclose(gv, gp[ridx] * w, rtol=1e-6) and np.allclose(gw[:, 0], (gp[ridx] * rgb).sum(1), rtol=1e-5, atol=1e-6)
    assert np.array_equal(gv, gv2) and np.allclose(gw2[:, 0] - gw[:, 0], gp[ridx][:, 2] * (rgb[:, 1] - rgb[:, 2]), atol=1e-5)


GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ref_*.npz")))


@pytest.mark.skipif(not GOLDEN, reason="reference-made fixtures not generated yet (tests/golden/make_ref_golden.py on a GPU)")
def test_oracle_matches_reference_made_fixtures():
    """Fixtures = outputs of the reference's own kernels (oracle/_ref) on seeded inputs; see make_ref_golden.py"""
    import golden.check_golden as cg
    for path in GOLDEN:
        cg.check(path, orc)
