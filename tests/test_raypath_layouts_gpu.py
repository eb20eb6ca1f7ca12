"""The ray path (csrc/volrender.cu, csrc/rayops.cu) on ragged, degenerate and multi-block layouts, through the C ABI.

Three layout families: ragged (lengths 0 .. 1023 with gaps between rays, and rays skipped because end > max_nr_samples), equal
(fixed_n 1, 16, 32, 33) and multi-block (1023 .. 8192 rays, and one set of more than 1024 * 1024 rays with 0-2 samples each). Every
output buffer carries NaN rows past N and R, and is NaN before the call, so a row the ABI does not name for a ray stays NaN.

  * against the serial C oracle, bit for bit: every index / start_end result and every serial-order float result, the importance
    samples with jitter off and on, the merge, the compaction and the occupancy sampler;
  * against the fp64 reference (oracle/raypath_fp64.py): the differentiable kernels and their backward, max|err| / max|ref| <= 1e-3
    and |err| <= EPS A element by element; `pytest -s` prints the worst err / bound ratio of each case;
  * ray locality: the importance samples of a ray do not change when every other ray's rows, the gaps between rays and the cdf
    scratch change.
"""
import numpy as np
import pytest
import torch

from oracle import rayops as orc
from oracle import raypath_fp64 as rf

pytestmark = pytest.mark.gpu
PAD = 37                                 # NaN sentinel rows past N and R
ST, INC = orc.PCG_STATE, orc.PCG_INC


@pytest.fixture(autouse=True)
def _device(cuda):
    """every test needs the H100 and the built library (skipped without a CUDA device)"""
    return cuda


def call(name, *args):
    from permuto_sdf_b200._lib import call as c
    return c(name, *args)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def N(t):
    return t.detach().cpu().numpy()


def nan_np(rows, cols):
    return np.full((rows + PAD, cols), np.nan, np.float32)


def nan_dev(rows, cols):
    return torch.full((rows + PAD, cols), float("nan"), device="cuda")


def bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape, what
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    bad = a != b
    assert not bad.any(), "%s: %d elements differ from the oracle (first at %s)" % (what, int(bad.sum()), np.argwhere(bad)[0])


def sentinel_kept(a, n, what):
    assert np.isnan(np.asarray(a)[n:]).all(), "%s: a row past the end was written" % what


# ------------------------------------------------------------------------------------------------ layouts
class Lay:
    def __init__(self, name, se, M, equal=False, fixed_n=0):
        self.name, self.se, self.M, self.equal, self.fixed_n = name, np.ascontiguousarray(se, np.int32), int(M), equal, fixed_n
        self.R = self.se.shape[0]
        if equal:
            s = np.arange(self.R) * fixed_n
            self.rng_se = np.stack([s, s + fixed_n], 1)
        else:
            self.rng_se = self.se.astype(np.int64)
        self.n = self.rng_se[:, 1] - self.rng_se[:, 0]
        self.skip = (self.rng_se[:, 1] > self.M) | (self.n == 0)
        self._dev, self._ref = None, None

    @property
    def se_dev(self):
        if self._dev is None:
            self._dev = T(self.se)
        return self._dev

    def rsp(self):
        return (self.R, self.M, self.se_dev, int(self.equal), int(self.fixed_n))

    def orsp(self):
        return (self.R, self.M, self.se, int(self.equal), int(self.fixed_n))

    def ref(self):
        if self._ref is None:
            self._ref = rf.layout(self.se, self.R, self.M, self.equal, self.fixed_n)
        return self._ref

    def owner(self):
        """ray index owning each of the M rows (-1: gap or skipped ray)"""
        own = np.full(self.M, -1, np.int64)
        for_rays = np.nonzero(~self.skip)[0]
        rows = np.concatenate([np.arange(self.rng_se[r, 0], self.rng_se[r, 1]) for r in for_rays]) if len(for_rays) else np.zeros(0, int)
        own[rows] = np.repeat(for_rays, self.n[for_rays])
        return own


def _multiblock(R, seed, max_len=70, skip_frac=0.01):
    rng = np.random.RandomState(seed)
    n = rng.randint(0, max_len + 1, R)
    gaps = rng.randint(0, 3, R)
    start = np.cumsum(gaps + n) - n
    se = np.stack([start, start + n], 1)
    M = int(se[-1, 1]) if R else 0
    sk = rng.rand(R) < skip_frac
    se[sk] = np.stack([se[sk, 0], np.full(sk.sum(), M + 5)], 1)
    return se, M


def _layouts():
    se, M = rf.ragged_layout(seed=0, copies=3)
    out = [Lay("ragged", se, M)]
    for fn in (1, 16, 32, 33):
        R = 300
        out.append(Lay("equal%d" % fn, np.zeros((R, 2), np.int32), R * fn - 2 * fn, True, fn))      # the last two rays are skipped
    for R in (1023, 1024, 1025, 4097, 8192):
        se, M = _multiblock(R, R)
        out.append(Lay("multi%d" % R, se, M))
    return out


LAYOUTS = _layouts()
IDS = [l.name for l in LAYOUTS]


def _inputs(lay, seed):
    rng = np.random.RandomState(seed)
    M, R = lay.M, lay.R
    own = lay.owner()
    d = dict(
        alpha=(0.6 + 0.4 * rng.rand(M, 1)).astype(np.float32),
        w=rng.rand(M, 1).astype(np.float32),
        vals=(rng.rand(M, 3) - 0.3).astype(np.float32),
        z=np.cumsum(rng.rand(M, 1) * 0.004 + 1e-4, 0).astype(np.float32) + 0.5,
        sdf=(0.3 - np.cumsum(rng.rand(M, 1) * 0.003, 0) % 0.6).astype(np.float32),
        rgb=rng.rand(M, 3).astype(np.float32),
        dt=(rng.rand(M, 1) * 0.004 + 1e-4).astype(np.float32),
        o=(rng.rand(R, 3) - 0.5).astype(np.float32),
        fixed_dt=(rng.rand(R, 1) * 0.004 + 1e-3).astype(np.float32),
        t_exit=(3.0 + rng.rand(R, 1)).astype(np.float32),
    )
    dr = rng.randn(R, 3)
    d["dirs"] = (dr / np.linalg.norm(dr, axis=1, keepdims=True)).astype(np.float32)
    scale = np.exp(rng.uniform(np.log(1.0), np.log(3e5), R)).astype(np.float32)       # early-outs anywhere along a ray, or none
    d["rad"] = (rng.rand(M, 1) * scale[np.maximum(own, 0)][:, None]).astype(np.float32)
    return d


def _ocall(name, *args):
    orc._call(name, *args)


def _gpu_cdf(lay, w):
    cdf = torch.zeros(lay.M, 1, device="cuda")
    call("psdf_vr_compute_cdf", *lay.rsp(), w, cdf)
    return cdf


def _normalised_cdf(lay, w):
    """per-ray normalised exclusive cdf of w (oracle arithmetic): a valid input for the importance sampler"""
    s_ray, s_smp = np.zeros((lay.R, 1), np.float32), np.ones((lay.M, 1), np.float32)
    _ocall("oracle_vr_sum_over_each_ray", *lay.orsp(), 1, w, s_ray, s_smp)
    wn = (w / np.maximum(s_smp, 1e-6)).astype(np.float32)
    cdf = np.zeros((lay.M, 1), np.float32)
    _ocall("oracle_vr_compute_cdf", *lay.orsp(), wn, cdf)
    return cdf


# ------------------------------------------------------------------------------------------------ oracle, bit for bit
@pytest.mark.parametrize("lay", LAYOUTS, ids=IDS)
def test_serial_kernels_bit_exact(lay):
    d = _inputs(lay, 1)
    M, R = lay.M, lay.R
    # transmittance
    gT, gbg = nan_dev(M, 1), nan_dev(R, 1)
    call("psdf_vr_cumprod_alpha2transmittance", *lay.rsp(), T(d["alpha"]), gT, gbg)
    eT, ebg = nan_np(M, 1), nan_np(R, 1)
    ebg[:R][lay.skip] = 1                     # the rows the ABI names for a skipped ray; the oracle leaves them to its caller
    _ocall("oracle_vr_cumprod_alpha2transmittance", *lay.orsp(), d["alpha"], eT, ebg)
    bits(N(gT), eT, "transmittance"); bits(N(gbg), ebg, "bg_transmittance")
    sentinel_kept(N(gT), M, "transmittance"); sentinel_kept(N(gbg), R, "bg_transmittance")
    assert (N(gbg)[:R][lay.skip] == 1).all()
    # integrate
    g, e = nan_dev(R, 3), nan_np(R, 3)
    e[:R][lay.skip] = 0
    call("psdf_vr_integrate_with_weights", *lay.rsp(), T(d["vals"]), T(d["w"]), g)
    _ocall("oracle_vr_integrate_with_weights", *lay.orsp(), d["vals"], d["w"], e)
    bits(N(g), e, "integrate")
    # sums, D = 1 (warp windows) and the per-channel lanes
    for D in (1, 2, 3, 32):
        v = np.random.RandomState(D).rand(M, D).astype(np.float32)
        gr, gs, er, es = nan_dev(R, D), nan_dev(M, D), nan_np(R, D), nan_np(M, D)
        er[:R][lay.skip] = 0
        call("psdf_vr_sum_over_each_ray", *lay.rsp(), D, T(v), gr, gs)
        _ocall("oracle_vr_sum_over_each_ray", *lay.orsp(), D, v, er, es)
        bits(N(gr), er, "sum_ray D=%d" % D); bits(N(gs), es, "sum_sample D=%d" % D)
        assert (N(gr)[:R][lay.skip] == 0).all()
        gg, eg = nan_dev(M, D), nan_np(M, D)
        gs_in = np.random.RandomState(D + 9).rand(M, D).astype(np.float32)
        gr_in = np.random.RandomState(D + 8).rand(R, D).astype(np.float32)
        call("psdf_vr_sum_over_each_ray_backward", *lay.rsp(), D, T(gr_in), T(gs_in), gg)
        _ocall("oracle_vr_sum_backward", *lay.orsp(), D, gr_in, gs_in, eg)
        bits(N(gg), eg, "sum backward D=%d" % D)
    # cumsum (forward / reverse), cdf, dt
    for inv in (0, 1):
        g, e = nan_dev(M, 1), nan_np(M, 1)
        call("psdf_vr_cumsum_over_each_ray", *lay.rsp(), T(d["w"]), inv, g)
        _ocall("oracle_vr_cumsum_over_each_ray", *lay.orsp(), d["w"], inv, e)
        bits(N(g), e, "cumsum inverse=%d" % inv)
    g, e = nan_dev(M, 1), nan_np(M, 1)
    call("psdf_vr_compute_cdf", *lay.rsp(), T(d["w"]), g)
    _ocall("oracle_vr_compute_cdf", *lay.orsp(), d["w"], e)
    bits(N(g), e, "cdf")
    for use in (0, 1):
        g, e = nan_dev(M, 1), nan_np(M, 1)
        call("psdf_vr_compute_dt", *lay.rsp(), use, T(d["t_exit"]), T(d["z"]), g)
        _ocall("oracle_vr_compute_dt", R, use, d["t_exit"], M, d["z"], lay.se, int(lay.equal), lay.fixed_n, e)
        bits(N(g), e, "compute_dt use_t_exit=%d" % use)
    # backward kernels
    cs = np.zeros((M, 1), np.float32)
    _ocall("oracle_vr_cumsum_over_each_ray", *lay.orsp(), (d["w"] * eT[:M]).astype(np.float32), 1, cs)
    g_bg = np.random.RandomState(5).rand(R, 1).astype(np.float32)
    g, e = nan_dev(M, 1), nan_np(M, 1)
    call("psdf_vr_cumprod_alpha2transmittance_backward", *lay.rsp(), T(g_bg), T(d["alpha"]), gbg[:R].contiguous(), T(cs), g)
    _ocall("oracle_vr_cumprod_backward", *lay.orsp(), g_bg, d["alpha"], ebg[:R], cs, e)
    bits(N(g), e, "cumprod backward")
    gp = (np.random.RandomState(6).rand(R, 3) - 0.5).astype(np.float32)
    for bug in (0, 1):
        gv, gw, ev, ew = nan_dev(M, 3), nan_dev(M, 1), nan_np(M, 3), nan_np(M, 1)
        call("psdf_vr_integrate_with_weights_backward", *lay.rsp(), T(gp), T(d["vals"]), T(d["w"]), bug, gv, gw)
        _ocall("oracle_vr_integrate_backward", *lay.orsp(), gp, d["vals"], d["w"], bug, ev, ew)
        bits(N(gv), ev, "integrate backward vals bug=%d" % bug); bits(N(gw), ew, "integrate backward w bug=%d" % bug)


@pytest.mark.parametrize("jitter", [0, 1])
@pytest.mark.parametrize("lay", LAYOUTS, ids=IDS)
def test_importance_sample_bit_exact(lay, jitter):
    d = _inputs(lay, 2)
    cdf = _normalised_cdf(lay, d["w"])
    for nr_imp in (16, 33, 70):                 # one window, lanes looping past 32, and past 64
        R = lay.R
        pos, dirs, z = nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 1)
        call("psdf_vr_importance_sample", *lay.rsp(), T(d["o"]), T(d["dirs"]), T(d["fixed_dt"]), T(d["z"]), T(cdf), nr_imp, ST, INC, jitter,
             pos, dirs, z)
        p = orc.Packed(R, lay.M)
        p.start_end, p.max_nr_samples, p.equal, p.fixed_n, p.z, p.fixed_dt = lay.se, lay.M, lay.equal, lay.fixed_n, d["z"], d["fixed_dt"]
        q = orc.vr_importance_sample(d["o"], d["dirs"], p, cdf, nr_imp, bool(jitter), ST, INC)
        n = R * nr_imp
        bits(N(z)[:n], q.z, "importance z nr_imp=%d" % nr_imp)
        bits(N(pos)[:n], q.pos, "importance pos nr_imp=%d" % nr_imp)
        bits(N(dirs)[:n], q.dirs, "importance dirs nr_imp=%d" % nr_imp)
        for a in (pos, dirs, z):
            sentinel_kept(N(a), n, "importance samples")
        gz = N(z)[:n, 0].reshape(R, nr_imp)
        dead = lay.skip | (lay.n == 1)
        assert (gz[dead] == -1).all() and (gz[~dead] >= 0).all()


def _separate_round(lay, d, nr_imp, jitter, inv_s=512.0, mult=1.5):
    """sdf2alpha -> clip -> cumprod(1 - a + 1e-7) -> w -> per-ray sum -> normalise -> cdf -> importance_sample, kernel by kernel"""
    M, R = lay.M, lay.R
    a = torch.zeros(M, 1, device="cuda")
    call("psdf_vr_sdf2alpha", *lay.rsp(), T(d["fixed_dt"]), T(d["dt"]), T(d["sdf"]), inv_s, 1, mult, a)
    a = a.clip(0.0, 1.0)
    Tt, bg = torch.zeros(M, 1, device="cuda"), torch.ones(R, 1, device="cuda")
    call("psdf_vr_cumprod_alpha2transmittance", *lay.rsp(), (1 - a + 1e-7).contiguous(), Tt, bg)
    w = (a * Tt).contiguous()
    sr, ss = torch.zeros(R, 1, device="cuda"), torch.zeros(M, 1, device="cuda")
    call("psdf_vr_sum_over_each_ray", *lay.rsp(), 1, w, sr, ss)
    w = (w / torch.clamp(ss, min=1e-6)).contiguous()
    cdf = _gpu_cdf(lay, w)
    pos, dirs, z = nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 1)
    call("psdf_vr_importance_sample", *lay.rsp(), T(d["o"]), T(d["dirs"]), T(d["fixed_dt"]), T(d["z"]), cdf, nr_imp, ST, INC, jitter,
         pos, dirs, z)
    return cdf, pos, dirs, z


def _fused_round(lay, d, nr_imp, jitter, scratch, inv_s=512.0, mult=1.5):
    R = lay.R
    cdf = torch.full((lay.M, 1), scratch, device="cuda")
    pos, dirs, z = nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 1)
    call("psdf_vr_importance_round", *lay.rsp(), T(d["o"]), T(d["dirs"]), T(d["fixed_dt"]), T(d["dt"]), T(d["z"]), T(d["sdf"]), inv_s, 1, mult,
         nr_imp, ST, INC, jitter, cdf, pos, dirs, z)
    return cdf, pos, dirs, z


@pytest.mark.parametrize("jitter", [0, 1])
@pytest.mark.parametrize("lay", LAYOUTS, ids=IDS)
def test_importance_round_equals_separate_kernels(lay, jitter):
    d = _inputs(lay, 3)
    own = lay.owner() >= 0
    for nr_imp in (16, 40):
        sc, sp, sd, sz = _separate_round(lay, d, nr_imp, jitter)
        fc, fp, fd, fz = _fused_round(lay, d, nr_imp, jitter, float("nan"))
        bits(N(fc)[own], N(sc)[own], "fused round cdf nr_imp=%d" % nr_imp)
        for a, b, nm in ((fp, sp, "pos"), (fd, sd, "dirs"), (fz, sz, "z")):
            bits(N(a), N(b), "fused round %s nr_imp=%d" % (nm, nr_imp))


def _perturb(lay, d, keep_rays, seed):
    """inputs where every row not owned by a ray in `keep_rays` (other rays, gaps) is replaced"""
    rng = np.random.RandomState(seed)
    own = lay.owner()
    other = ~np.isin(own, np.nonzero(keep_rays)[0])
    e = dict(d)
    for k in ("z", "sdf", "dt", "w", "alpha"):
        v = d[k].copy()
        v[other] = (rng.rand(int(other.sum()), v.shape[1]) * 3 - 1).astype(np.float32)
        e[k] = v
    return e


LOCALITY = [l for l in LAYOUTS if l.name in ("ragged", "equal1", "equal16", "equal33", "multi1025")]


@pytest.mark.parametrize("lay", LOCALITY, ids=[l.name for l in LOCALITY])
def test_ray_locality(lay):
    """the importance samples of every even (then odd) ray are bit-identical when everything outside that ray changes; one-sample
    rays, whose cdf search would reach into the previous ray's rows, included"""
    d = _inputs(lay, 4)
    R, nr_imp = lay.R, 40
    rays = np.arange(R)
    for parity in (0, 1):
        keep = (rays % 2) == parity
        e = _perturb(lay, d, keep, 10 + parity)
        cdf_d = _normalised_cdf(lay, d["w"])
        cdf_e = _normalised_cdf(lay, e["w"])
        cdf_e[~np.isin(lay.owner(), np.nonzero(keep)[0])] = np.nan
        kz = np.repeat(keep, nr_imp)
        for jitter in (0, 1):
            outs = []
            for dd, cdf in ((d, cdf_d), (e, cdf_e)):
                pos, dirs, z = nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 3), nan_dev(R * nr_imp, 1)
                call("psdf_vr_importance_sample", *lay.rsp(), T(dd["o"]), T(dd["dirs"]), T(dd["fixed_dt"]), T(dd["z"]), T(cdf), nr_imp, ST,
                     INC, jitter, pos, dirs, z)
                outs.append((N(pos)[:R * nr_imp][kz], N(z)[:R * nr_imp][kz]))
            for (a, b), nm in zip(zip(*outs), ("pos", "z")):
                assert np.isfinite(a).all(), "importance_sample %s: non-finite samples" % nm
                bits(a, b, "importance_sample %s of the kept rays (parity %d, jitter %d)" % (nm, parity, jitter))
            outs = []
            for dd, scratch in ((d, 0.25), (e, float("nan"))):
                cdf, pos, dirs, z = _fused_round(lay, dd, nr_imp, jitter, scratch)
                outs.append((N(pos)[:R * nr_imp][kz], N(z)[:R * nr_imp][kz]))
            for (a, b), nm in zip(zip(*outs), ("pos", "z")):
                assert np.isfinite(a).all(), "importance_round %s: non-finite samples" % nm
                bits(a, b, "importance_round %s of the kept rays (parity %d, jitter %d)" % (nm, parity, jitter))


# ------------------------------------------------------------------------------------------------ fp64 reference
@pytest.mark.parametrize("lay", LAYOUTS, ids=IDS)
def test_differentiable_kernels_against_fp64(lay):
    d = _inputs(lay, 5)
    M, R = lay.M, lay.R
    L = lay.ref()
    rep = {}
    rng = np.random.RandomState(8)
    a = d["alpha"].copy()
    a[rng.rand(M) < 0.003] = 3e-7                 # rays with a factor below 1e-6: the division form is not the derivative there
    gT, gbg = nan_dev(M, 1), nan_dev(R, 1)
    call("psdf_vr_cumprod_alpha2transmittance", *lay.rsp(), T(a), gT, gbg)
    ref = rf.cumprod(L, a)
    rf.check("T", N(gT)[:M, 0], ref["T"], ref["A_T"], ref["rows"], rep)
    rf.check("bg_T", N(gbg)[:R, 0], ref["bg"], ref["A_bg"], report=rep)
    g_T, g_bg = T(rng.rand(M, 1).astype(np.float32)), T(rng.rand(R, 1).astype(np.float32))
    cs = torch.zeros(M, 1, device="cuda")
    call("psdf_vr_cumsum_over_each_ray", *lay.rsp(), (g_T * gT[:M]).contiguous(), 1, cs)
    ga = nan_dev(M, 1)
    call("psdf_vr_cumprod_alpha2transmittance_backward", *lay.rsp(), g_bg, T(a), gbg[:R].contiguous(), cs, ga)
    ref = rf.cumprod_backward(L, a, N(g_T), N(g_bg))
    rf.check("cumprod backward", N(ga)[:M, 0], ref["g_alpha"], ref["A"], ref["rows"] & rf.rows_of(L, M, ref["exact_rays"]), rep)
    g = nan_dev(R, 3)
    call("psdf_vr_integrate_with_weights", *lay.rsp(), T(d["vals"]), T(d["w"]), g)
    ref = rf.integrate(L, d["vals"], d["w"])
    rf.check("integrate", N(g)[:R], ref["out"], ref["A"], report=rep)
    gp = (rng.rand(R, 3) - 0.5).astype(np.float32)
    gv, gw = nan_dev(M, 3), nan_dev(M, 1)
    call("psdf_vr_integrate_with_weights_backward", *lay.rsp(), T(gp), T(d["vals"]), T(d["w"]), 0, gv, gw)
    ref = rf.integrate_backward(L, gp, d["vals"], d["w"])
    rf.check("integrate backward vals", N(gv)[:M], ref["g_vals"], ref["A_vals"], ref["rows"], rep)
    rf.check("integrate backward w", N(gw)[:M, 0], ref["g_w"], ref["A_w"], ref["rows"], rep)
    for D in (1, 3):
        v = (rng.rand(M, D) - 0.3).astype(np.float32)
        sr, ss = nan_dev(R, D), nan_dev(M, D)
        call("psdf_vr_sum_over_each_ray", *lay.rsp(), D, T(v), sr, ss)
        ref = rf.sum_over_each_ray(L, v)
        rf.check("sum ray D=%d" % D, N(sr)[:R], ref["sum_ray"], ref["A_ray"], report=rep)
        rf.check("sum sample D=%d" % D, N(ss)[:M], ref["sum_sample"], ref["A_sample"], ref["rows"], rep)
        gr, gs = rng.rand(R, D).astype(np.float32), rng.rand(M, D).astype(np.float32)
        gg = nan_dev(M, D)
        call("psdf_vr_sum_over_each_ray_backward", *lay.rsp(), D, T(gr), T(gs), gg)
        ref = rf.sum_over_each_ray_backward(L, gr, gs)
        rf.check("sum backward D=%d" % D, N(gg)[:M], ref["g_vals"], ref["A"], ref["rows"], rep)
    # NeRF render and its backward, the T < 1e-4 early-out landing anywhere in the warp windows
    pr, dp, bg, w = nan_dev(R, 3), nan_dev(R, 1), nan_dev(R, 1), nan_dev(M, 1)
    call("psdf_vr_volume_render_nerf", *lay.rsp(), T(d["rgb"]), T(d["rad"]), T(d["z"]), T(d["dt"]), pr, dp, bg, w)
    gpr, gbt = (rng.rand(R, 3) - 0.5).astype(np.float32), (rng.rand(R, 1) - 0.5).astype(np.float32)
    grgb, grad = nan_dev(M, 3), nan_dev(M, 1)
    call("psdf_vr_volume_render_nerf_backward", *lay.rsp(), T(gpr), T(gbt), pr[:R].contiguous(), bg[:R].contiguous(), T(d["rgb"]),
         T(d["rad"]), T(d["dt"]), grgb, grad)
    ref = rf.volume_render_nerf(L, d["rgb"], d["rad"], d["z"], d["dt"], gpr, gbt)
    ok = ~ref["ambiguous"]
    okr = ref["written"] & rf.rows_of(L, M, ok)
    rf.check("nerf rgb", N(pr)[:R], ref["pred"], ref["A_pred"], ok, rep)
    rf.check("nerf depth", N(dp)[:R, 0], ref["depth"], ref["A_depth"], ok, rep)
    rf.check("nerf bg_T", N(bg)[:R, 0], ref["bg"], ref["A_bg"], ok, rep)
    rf.check("nerf w", N(w)[:M, 0], ref["w"], ref["A_w"], okr, rep)
    rf.check("nerf g_rgb", N(grgb)[:M], ref["g_rgb"], ref["A_g_rgb"], okr, rep)
    rf.check("nerf g_radiance", N(grad)[:M, 0], ref["g_rad"], ref["A_g_rad"], okr, rep)
    # rows after the early-out, of skipped rays and past the end keep the sentinel
    unwritten = ~ref["written"].numpy() & rf.rows_of(L, M, ok).numpy()
    for a, nm in ((w, "w"), (grgb, "g_rgb"), (grad, "g_radiance")):
        assert np.isnan(N(a)[:M][unwritten]).all(), "nerf %s: a row after the early-out was written" % nm
        sentinel_kept(N(a), M, "nerf " + nm)
    sk = lay.skip
    assert (N(bg)[:R][sk] == 1).all() and (N(pr)[:R][sk] == 0).all() and (N(dp)[:R][sk] == 0).all()
    print("\n%s: worst err/bound %s; %d ambiguous early-outs" % (lay.name, ", ".join("%s %.3g" % kv for kv in sorted(rep.items())),
                                                                   int((~ok).sum())))


# ------------------------------------------------------------------------------------------------ merge, compaction
def _merge_case(u_lens, imp_n, seed, tie_frac=0.05):
    rng = np.random.RandomState(seed)
    R = len(u_lens)
    n = np.asarray(u_lens)
    start = np.cumsum(n + 2) - n
    se = np.stack([start, start + n], 1).astype(np.int32)
    M = int(se[-1, 1]) + 3 if R else 1
    u_z = np.full((M, 1), np.nan, np.float32)
    i_z = np.zeros((R * imp_n, 1), np.float32)
    for r in range(R):                            # sorted samples per ray; some importance z equal to a uniform z (the tie rule)
        u = np.sort(rng.rand(n[r])).astype(np.float32)
        u_z[se[r, 0]:se[r, 1], 0] = u
        iz = np.sort(rng.rand(imp_n)).astype(np.float32)
        if n[r]:
            tie = rng.rand(imp_n) < tie_frac
            iz[tie] = u[rng.randint(0, n[r], int(tie.sum()))]
            iz.sort()
        i_z[r * imp_n:(r + 1) * imp_n, 0] = iz
    return se, M, u_z, i_z


def _merge(se, M, u_z, i_z, imp_n, seed):
    rng = np.random.RandomState(seed)
    R = se.shape[0]
    o, dr = (rng.rand(R, 3) - 0.5).astype(np.float32), (rng.rand(R, 3) - 0.5).astype(np.float32)
    tx = (0.8 + 0.4 * rng.rand(R, 1)).astype(np.float32)
    fdt = (rng.rand(R, 1) * 0.01).astype(np.float32)
    u_sdf, i_sdf = rng.rand(M, 1).astype(np.float32), rng.rand(R * imp_n, 1).astype(np.float32)
    c_max = M + R * imp_n
    nb = (R + 1023) // 1024
    ws = torch.full((R + nb + 1,), -7, dtype=torch.int32, device="cuda")
    gp, gd, gz, gdt, gs = nan_dev(c_max, 3), nan_dev(c_max, 3), nan_dev(c_max, 1), nan_dev(c_max, 1), nan_dev(c_max, 1)
    gf, gse = nan_dev(R, 1), torch.full((R + PAD, 2), -7, dtype=torch.int32, device="cuda")
    call("psdf_vr_combine_uniform_samples_with_imp", R, M, T(se), 0, 0, T(o), T(dr), T(tx), T(fdt), T(u_z), T(u_sdf), 1, imp_n, T(i_z),
         T(i_sdf), 1, c_max, ws, gp, gd, gz, gdt, gs, gf, gse)
    p = orc.Packed(R, M)
    p.start_end, p.z, p.sdf, p.fixed_dt, p.has_sdf = se, u_z, u_sdf, fdt, True
    q = orc.Packed(R, R * imp_n)
    q.z, q.sdf, q.has_sdf, q.fixed_n, q.equal = i_z, i_sdf, True, imp_n, True
    e = orc.vr_combine(o, dr, tx, p, q)
    total = int(N(ws)[R + nb])
    assert total == e.cur
    bits(N(gse)[:R], e.start_end, "merged start_end")
    assert (N(gse)[R:] == -7).all()
    bits(N(gf)[:R], e.fixed_dt, "merged fixed_dt")
    for a, b, nm in ((gz, e.z, "z"), (gdt, e.dt, "dt"), (gp, e.pos, "pos"), (gd, e.dirs, "dirs"), (gs, e.sdf, "sdf")):
        got = N(a)
        assert np.isfinite(got[:total]).all(), "merged %s: a slot of a merged ray was not written" % nm
        bits(got[:total], b[:total], "merged " + nm)
        sentinel_kept(got, total, "merged " + nm)
    zz = N(gz)[:total, 0]
    for s, t in e.start_end[(e.start_end[:, 1] - e.start_end[:, 0]) > 1000]:
        assert (np.diff(zz[s:t]) >= 0).all()
    return e


@pytest.mark.parametrize("imp_n", [16, 48])
def test_merge_long_rays(imp_n):
    """merged lengths 1023, 1024, 1025, 2048 and 4097 beside short, one-sample and empty rays"""
    targets = [1023, 1024, 1025, 2048, 4097]
    u_lens = [t - imp_n for t in targets] + [5, 64, 1, 0, 2, 33] + [t - imp_n for t in targets[::-1]]
    se, M, u_z, i_z = _merge_case(u_lens, imp_n, imp_n)
    e = _merge(se, M, u_z, i_z, imp_n, 1)
    n = e.start_end[:, 1] - e.start_end[:, 0]
    assert sorted(set(n.tolist())) == sorted(set([0] + [l + imp_n for l in u_lens if l > 1]))


MULTI_R = [1023, 1024, 1025, 4097, 8192, 1024 * 1024 + 3001]


@pytest.mark.parametrize("R", MULTI_R)
def test_multiblock_scans(R):
    """the block-local scans and the scan of the block sums (its chunk loop past 1024 blocks) of the merge and the compaction"""
    rng = np.random.RandomState(R % 1000)
    big = R > 1024 * 1024
    n = rng.randint(0, 3, R) if big else rng.randint(0, 40, R)
    start = np.cumsum(n + rng.randint(0, 2, R)) - n
    se = np.stack([start, start + n], 1).astype(np.int32)
    M = int(se[-1, 1]) + 1
    imp_n = 2 if big else 8
    u_z = np.zeros((M, 1), np.float32)
    u_z[:, 0] = np.arange(M, dtype=np.float32) * 1e-6 + rng.rand(M).astype(np.float32) * 1e-7
    i_z = np.sort(rng.rand(R, imp_n).astype(np.float32) * M * 1e-6, 1).reshape(-1, 1)
    _merge(se, M, u_z, i_z, imp_n, 2)
    # compaction of the same packed set
    pos, dirs = rng.rand(M, 3).astype(np.float32), rng.rand(M, 3).astype(np.float32)
    z, dt, sdf, fdt = (rng.rand(M, 1).astype(np.float32) for _ in range(4))
    fdt = rng.rand(R, 1).astype(np.float32)
    wsb = call("psdf_packed_compact_workspace_bytes", R)
    ws = torch.full((wsb // 4,), -7, dtype=torch.int32, device="cuda")
    call("psdf_packed_compact_scan", R, T(se), ws)
    total = int(n.sum())
    assert int(N(ws)[R + (R + 1023) // 1024]) == total
    o = [nan_dev(total, c) for c in (3, 3, 1, 1, 1)]
    of, ose = nan_dev(R, 1), torch.full((R + PAD, 2), -7, dtype=torch.int32, device="cuda")
    call("psdf_packed_compact_copy", R, T(pos), None, T(dirs), T(z), T(dt), T(sdf), T(fdt), T(se), ws, o[0], None, o[1], o[2], o[3], o[4],
         of, ose)
    p = orc.Packed(R, M)
    p.pos, p.dirs, p.z, p.dt, p.sdf, p.fixed_dt, p.start_end, p.has_sdf = pos, dirs, z, dt, sdf, fdt, se, True
    q = orc.packed_compact(p)
    assert q.cur == total
    bits(N(ose)[:R], q.start_end, "compacted start_end")
    bits(N(of)[:R], q.fixed_dt, "compacted fixed_dt")
    for a, b, nm in zip(o, (q.pos, q.dirs, q.z, q.dt, q.sdf), ("pos", "dirs", "z", "dt", "sdf")):
        bits(N(a)[:total], b[:total], "compacted " + nm)
        sentinel_kept(N(a), total, "compacted " + nm)


# ------------------------------------------------------------------------------------------------ occupancy sampler
def _box_rays(R, extent, trans, seed, kinds):
    """rays through the grid's box [trans - extent/2, trans + extent/2]: random, axis-aligned, grazing a face, t_entry == t_exit"""
    rng = np.random.RandomState(seed)
    c, h = np.asarray(trans, np.float64), extent / 2
    o = c + (rng.rand(R, 3) - 0.5) * extent * 3
    tgt = c + (rng.rand(R, 3) - 0.5) * extent * 0.8
    d = tgt - o
    k = 0
    if "axis" in kinds:
        for ax in range(3):
            for sgn in (1, -1):
                for j in range(4):
                    o[k] = c + (rng.rand(3) - 0.5) * extent * 0.9
                    if j == 0:
                        o[k] = c + np.round((o[k] - c) * 64) / 64       # on voxel boundaries
                    o[k, ax] = c[ax] - sgn * h * 1.5
                    d[k] = 0
                    d[k, ax] = sgn
                    k += 1
    if "graze" in kinds:
        for j in range(8):
            o[k] = c + (rng.rand(3) - 0.5) * extent * 0.9
            o[k, j % 3] = c[j % 3] + (h if j % 2 else -h)                   # in a face's plane
            d[k] = rng.randn(3)
            d[k, j % 3] = 0
            k += 1
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    o32, d32 = o.astype(np.float32), d.astype(np.float32)
    od, dd = o32.astype(np.float64), d32.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        t0 = (c - h - od) / dd
        t1 = (c + h - od) / dd
    tn = np.nan_to_num(np.minimum(t0, t1), nan=-np.inf).max(1)
    tf = np.nan_to_num(np.maximum(t0, t1), nan=np.inf).min(1)
    te, tx = np.maximum(tn, 0), np.maximum(tf, 0)
    miss = te >= tx
    te[miss] = tx[miss] = 0
    # an entry point on a face at the upper end of an axis lies outside the grid (the reference's voxel lookup), so the march ends
    # before it starts: most random rays enter slightly inside the box, a quarter exactly on its face
    inner = (np.arange(R) >= k) & (np.arange(R) % 4 != 0)
    te[inner] += 1e-3 * (tx[inner] - te[inner])
    if "flat" in kinds:
        te[k:k + 6] = tx[k:k + 6] = ((te[k:k + 6] + tx[k:k + 6]) / 2)        # t_entry == t_exit
    return o32, d32, te.astype(np.float32)[:, None], tx.astype(np.float32)[:, None]


def _occ(V, kind, seed):
    if kind == "full":
        return np.ones(V ** 3, np.uint8)
    rng = np.random.RandomState(seed)
    if kind == "dense":
        return (rng.rand(V ** 3) < 0.85).astype(np.uint8)
    return (rng.rand(V ** 3) < 0.3).astype(np.uint8)


OCC_CASES = [
    # name, V, extent, trans, occupancy, min_dist, max_per_ray, rays, kinds
    ("v512_full_maxsteps", 512, 1.0, (0, 0, 0), "full", 1e-4, 6000, 48, ()),
    ("v512_dense_steps", 512, 1.0, (0, 0, 0), "dense", 2e-4, 6000, 48, ()),
    ("v256_translated", 256, 2.5, (0.3, -0.2, 0.1), "sparse", 4e-3, 700, 200, ("axis", "graze", "flat")),
    ("v256_cap_in_window", 256, 2.5, (0.3, -0.2, 0.1), "sparse", 1e-4, 45, 200, ("axis", "graze", "flat")),
    ("v128_cap_77", 128, 1.0, (0, 0, 0), "dense", 1e-4, 77, 200, ("axis", "graze")),
]


@pytest.mark.parametrize("jitter", [0, 1])
@pytest.mark.parametrize("case", OCC_CASES, ids=[c[0] for c in OCC_CASES])
def test_occupancy_sampler_edges(case, jitter):
    name, V, extent, trans, kind, min_dist, mpr, R, kinds = case
    o, d, te, tx = _box_rays(R, extent, trans, V, kinds)
    occ = _occ(V, kind, V + 1)
    M = R * mpr
    pos, dirs, z, dt = nan_dev(M, 3), nan_dev(M, 3), nan_dev(M, 1), nan_dev(M, 1)
    fdt, se, cur = nan_dev(R, 1), torch.full((R + PAD, 2), -7, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    call("psdf_occ_compute_samples_in_occupied_regions", R, V, extent, trans, T(o), T(d), T(te), T(tx), T(occ), min_dist, mpr, M, ST, INC,
         jitter, 1, pos, dirs, z, dt, fdt, se, cur)
    e = orc.occ_samples_in_occupied_regions(V, extent, trans, o, d, te, tx, occ, min_dist, mpr, bool(jitter), ST, INC)
    gse = N(se)
    bits(gse[:R], e.start_end, "start_end")
    assert (gse[R:] == -7).all()
    assert int(N(cur)[0]) == e.cur
    bits(N(fdt)[:R], e.fixed_dt, "ray_fixed_dt")
    rows = np.zeros(M, bool)
    for s, t in e.start_end:
        rows[s:t] = True
    for a, b, nm in ((z, e.z, "z"), (dt, e.dt, "dt"), (pos, e.pos, "pos"), (dirs, e.dirs, "dirs")):
        bits(N(a)[:M][rows], b[rows], nm)
        sentinel_kept(N(a), M, nm)
    n = e.start_end[:, 1] - e.start_end[:, 0]
    if "maxsteps" in name:
        assert n.max() == 4096, "the march should stop at kMaxSteps"
    if "steps" in name:
        assert (n > 2000).any()
    if "cap" in name:
        assert (n == mpr).any() and (n % 32 != 0).any()
    print("\n%s jitter=%d: %d rays with samples, longest %d" % (name, jitter, int((n > 0).sum()), int(n.max())))
