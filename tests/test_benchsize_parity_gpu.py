"""Ray-path parity at the sizes bench.py runs (the other ray-path tests use V = 128 / 64 samples): 256^3 occupancy grid, 512 rays,
96 grid samples per ray at min distance 1e-4, then the two importance-sampling rounds with 16 samples each (128 samples per ray in
total), jitter off and on. Ours (through the `permuto_sdf` mirror / C ABI) against what the reference's own kernels compute on the same
seeded inputs (tests/golden/benchsize_reference.npz, generator: tests/golden/make_benchsize_golden.py) and, for the grid samples, against the C
oracle: per-ray sample counts, z, dt and positions must be bit-identical."""
import os

import numpy as np
import pytest
import torch

import scenes
from oracle import rayops as orc

pytestmark = pytest.mark.gpu
V, R, MAX_PER_RAY, NR_IMP, MIN_DIST = 256, 512, 96, 16, 1e-4
RAY_STEP = 16                 # the fixture keeps the samples of every RAY_STEP-th ray (all per-ray counts)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "benchsize_reference.npz")


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def scene(cuda):
    from permuto_sdf import OccupancyGrid, Sphere
    o, d = scenes.make_rays(R, seed=5, miss_fraction=0.05)
    values, occ = scenes.analytic_occupancy(V)
    grid = OccupancyGrid(V, 1.0, [0, 0, 0])
    grid.set_grid_values(T(values))
    grid.set_grid_occupancy(T(occ.astype(np.uint8)).bool())
    return dict(o=o, d=d, occ=occ.astype(np.uint8), grid=grid, sphere=Sphere(scenes.SPHERE_RADIUS, [0, 0, 0]))


def _per_ray_equal(se_a, arrs_a, se_b, arrs_b, what):
    assert np.array_equal(se_a[:, 1] - se_a[:, 0], se_b[:, 1] - se_b[:, 0]), what + ": per-ray sample counts differ"
    for (s, e), (rs, re) in zip(se_a, se_b):
        for a, b in zip(arrs_a, arrs_b):
            assert np.array_equal(a[s:e], b[rs:re]), what + ": samples not bit-identical"


def _subset(start_end, arrays):
    """per-ray counts of all rays, the samples of rays 0, RAY_STEP, ... concatenated in ray order (the fixture's layout)"""
    se = np.asarray(start_end)
    keep = [(s, e) for i, (s, e) in enumerate(se) if i % RAY_STEP == 0]
    return (se[:, 1] - se[:, 0]).astype(np.int32), [np.concatenate([a[s:e] for s, e in keep] + [a[:0]], 0) for a in arrays]


def _equal_to_fixture(G, prefix, start_end, arrays, what):
    n, got = _subset(start_end, arrays)
    assert np.array_equal(n, G[prefix + ".n"]), what + ": per-ray sample counts differ"
    for name, a in zip(("z", "dt", "pos"), got):
        assert np.array_equal(a, G[prefix + "." + name]), what + ": samples not bit-identical (%s)" % name


@pytest.mark.parametrize("jitter", [False, True])
def test_grid_sampling_and_importance_rounds_at_bench_size(scene, jitter):
    from permuto_sdf import OccupancyGrid, VolumeRendering
    G = dict(np.load(GOLDEN))
    key = "j%d" % int(jitter)
    # the random streams start from the generators' initial state, like the fixture's
    for rng in (OccupancyGrid.m_rng, VolumeRendering.m_rng):
        rng.to_host()
        rng.state, rng.inc = type(rng)().state, type(rng)().inc
    o, d = T(scene["o"]), T(scene["d"])
    _, te, _, tx, _ = scene["sphere"].ray_intersection(o, d)
    st, inc = OccupancyGrid.m_rng.state, OccupancyGrid.m_rng.inc
    uni = scene["grid"].compute_samples_in_occupied_regions(o, d, te, tx, MIN_DIST, MAX_PER_RAY, jitter)
    se = N(uni.ray_start_end_idx)
    assert (se[:, 1] - se[:, 0]).max() == MAX_PER_RAY, "the bench scene fills the per-ray budget"
    # (a) the C oracle
    exp = orc.occ_samples_in_occupied_regions(V, 1.0, [0, 0, 0], scene["o"], scene["d"], N(te), N(tx), scene["occ"], MIN_DIST, MAX_PER_RAY, jitter, st, inc)
    _per_ray_equal(se, [N(uni.samples_z), N(uni.samples_dt), N(uni.samples_pos)], exp.start_end, [exp.z, exp.dt, exp.pos], "grid samples vs C oracle")
    # (b) the reference kernels
    _equal_to_fixture(G, key + ".grid", se, [N(uni.samples_z), N(uni.samples_dt), N(uni.samples_pos)], "grid samples vs reference kernel")
    # importance sampling on the analytic SDF (identical sdf values on both sides), two rounds like sdf_utils.py:383-423
    ours = uni.compact_to_valid_samples()

    def sdf_of(pos):
        return (torch.sqrt((pos * pos).sum(1, keepdim=True)) - scenes.OBJECT_RADIUS).contiguous()

    for rnd, mult in enumerate((1.0, 2.0)):
        so = sdf_of(ours.samples_pos)
        ours.set_sdf(so)
        # ours: the fused round (one launch); the fixture holds the chain of reference kernels
        imp_o = VolumeRendering.importance_round(o, d, ours, so, 512.0, True, mult, NR_IMP, jitter)
        assert np.array_equal(N(imp_o.samples_z).reshape(R, NR_IMP)[::RAY_STEP], G["%s.imp%d.z" % (key, rnd)]), \
            "importance samples (round %d) differ from the reference kernels" % rnd
        imp_o.set_sdf(sdf_of(imp_o.samples_pos))
        ours = VolumeRendering.combine_uniform_samples_with_imp(o, d, tx, ours, imp_o).compact_to_valid_samples()
        _equal_to_fixture(G, "%s.merged%d" % (key, rnd), N(ours.ray_start_end_idx), [N(ours.samples_z), N(ours.samples_dt), N(ours.samples_pos)],
                          "merged samples after round %d" % rnd)
    n = N(ours.ray_start_end_idx)
    assert (n[:, 1] - n[:, 0]).max() == MAX_PER_RAY + 2 * NR_IMP, "128 samples per ray, the bench configuration"
