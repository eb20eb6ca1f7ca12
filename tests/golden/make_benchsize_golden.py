"""Generate tests/golden/benchsize_reference.npz: what the reference's own kernels (oracle/_ref/libpsdf_ref_gpu.so, built by
oracle/ref_shim/Makefile from a checkout of the original project) compute for the ray path at the sizes bench.py runs, on the
seeded scene of tests/test_benchsize_parity_gpu.py (256^3 occupancy grid, 512 rays, 96 grid samples per ray, two importance rounds of
16 samples, jitter off and on). Run on a GPU: `python tests/golden/make_benchsize_golden.py`.

Per-ray sample counts are stored for every ray; the samples themselves (z, dt, position; importance z) for every RAY_STEP-th ray, so
that the file stays small. The random streams start from the generators' initial state (as in a fresh process).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "compat")]
import scenes  # noqa: E402
from oracle import ref_gpu as ref  # noqa: E402

V, R, MAX_PER_RAY, NR_IMP, MIN_DIST = 256, 512, 96, 16, 1e-4
RAY_STEP = 16
OUT = os.path.join(HERE, "benchsize_reference.npz")


def N(t):
    return t.detach().cpu().numpy()


def subset(start_end, arrays):
    """per-ray counts of all rays, the samples of rays 0, RAY_STEP, 2 RAY_STEP, ... concatenated in ray order"""
    se = np.asarray(start_end)
    keep = [(s, e) for i, (s, e) in enumerate(se) if i % RAY_STEP == 0]
    return (se[:, 1] - se[:, 0]).astype(np.int32), [np.concatenate([a[s:e] for s, e in keep] + [a[:0]], 0) for a in arrays]


def sdf_of(pos):
    return (torch.sqrt((pos * pos).sum(1, keepdim=True)) - scenes.OBJECT_RADIUS).contiguous()


def main():
    from permuto_sdf import OccupancyGrid, VolumeRendering
    assert ref.available(), "oracle/_ref/libpsdf_ref_gpu.so missing: build it with PERMUTO_SDF_REFERENCE set"
    o_np, d_np = scenes.make_rays(R, seed=5, miss_fraction=0.05)
    values, occ = scenes.analytic_occupancy(V)
    o, d = torch.from_numpy(o_np).cuda(), torch.from_numpy(d_np).cuda()
    occ_t = torch.from_numpy(occ.astype(np.uint8)).cuda().bool()
    G = {}
    for jitter in (False, True):
        key = "j%d" % int(jitter)
        rng_grid, rng_vr = type(OccupancyGrid.m_rng)(), type(VolumeRendering.m_rng)()     # initial generator states
        _, te, _, tx, _ = ref.sphere_ray_intersection(scenes.SPHERE_RADIUS, [0, 0, 0], o, d)
        theirs = ref.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], o, d, te, tx, occ_t, MIN_DIST, MAX_PER_RAY, jitter, rng_grid.state,
                                                     rng_grid.inc)
        G[key + ".grid.n"], (G[key + ".grid.z"], G[key + ".grid.dt"], G[key + ".grid.pos"]) = subset(
            N(theirs.start_end), [N(theirs.z), N(theirs.dt), N(theirs.pos)])
        theirs = theirs.compact()
        for rnd, mult in enumerate((1.0, 2.0)):
            sr = sdf_of(theirs.pos)
            theirs.sdf, theirs.has_sdf = sr, True
            a = ref.vr_sdf2alpha(theirs, sr, 512.0, True, mult).clip(0.0, 1.0)
            Tr, _ = ref.vr_cumprod(theirs, 1 - a + 1e-7)
            w = a * Tr
            _, wsum = ref.vr_sum(theirs, w)
            w = w / torch.clamp(wsum, min=1e-6)
            cdf = ref.vr_cdf(theirs, w)
            imp_r = ref.vr_importance_sample(o, d, theirs, cdf, NR_IMP, jitter, rng_vr.state, rng_vr.inc)
            if jitter:
                rng_vr.advance()              # the jittered importance round advances the class generator once
            G["%s.imp%d.z" % (key, rnd)] = N(imp_r.z).reshape(R, NR_IMP)[::RAY_STEP].copy()
            imp_r.sdf, imp_r.has_sdf = sdf_of(imp_r.pos), True
            theirs = ref.vr_combine(o, d, tx, theirs, imp_r).compact()
            n, (z, dt, pos) = subset(N(theirs.start_end), [N(theirs.z), N(theirs.dt), N(theirs.pos)])
            G["%s.merged%d.n" % (key, rnd)], G["%s.merged%d.z" % (key, rnd)] = n, z
            G["%s.merged%d.dt" % (key, rnd)], G["%s.merged%d.pos" % (key, rnd)] = dt, pos
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    np.savez_compressed(out, **G)
    print("wrote", out, os.path.getsize(out), "bytes,", len(G), "arrays; gpu:", torch.cuda.get_device_name(0))


if __name__ == "__main__":
    main()
