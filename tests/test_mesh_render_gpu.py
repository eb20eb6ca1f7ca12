"""Mesh.first_hit and Mesh.render on the GPU: first hits equal the brute-force oracle (tests/first_hit_oracle.py) bit for bit on the scenes of
test_mesh_raycast_gpu.py, render outputs equal its shade of the first hits of PermutoSDF.rays_from_reel_indices' rays bit for bit, a
rendered marching-cubes sphere agrees with bench.analytic_reel's analytic one, the refusals, and a torus trained from its own renders."""
import math

import numpy as np
import pytest
import torch

import mesh_checks as C
import first_hit_oracle as FH
from permuto_sdf_b200.cameras import TensorReel, sphere_cameras
from permuto_sdf_b200.mesh import RENDER_OUTPUTS, Mesh, marching_cubes
from test_mesh_raycast_gpu import box_mesh, cu, floor_grid, mc_mesh, rand_dirs, rotation, two_spheres

pytestmark = pytest.mark.gpu

# the end-to-end budget and its bars (test_a_torus_trained_from_its_renders)
STEPS = 1000
PSNR_MIN = 13.5
CHAMFER_MAX = 0.025


def check(V, F, o, d, tnear=0.0, tfar=math.inf, expect_some=True):
    m = Mesh(cu(V), cu(np.asarray(F).reshape(-1, 3), torch.int32))
    t, f, b = (x.cpu().numpy() for x in m.first_hit(cu(o), cu(d), tnear, tfar))
    rt, rf, rb = FH.first_hit(V, F, o, d, np.float32(tnear), tfar)
    bad = np.flatnonzero(f != rf)
    assert bad.size == 0, (bad.size, bad[:10], f[bad[:3]], rf[bad[:3]], o[bad[:3]], d[bad[:3]])
    assert np.array_equal(t.view(np.int32), rt.view(np.int32)), "t differs"
    assert np.array_equal(b.view(np.int32), rb.view(np.int32)), "bary differs"
    if expect_some:
        assert 0 < (rf >= 0).sum() < rf.size
    return rt, rf, rb


# ------------------------------------------------------------------------------------------------ first_hit == brute force
@pytest.mark.parametrize("seed", [0, 1])
def test_random_soups(cuda, seed):
    rng = np.random.default_rng(seed)
    F = 1500
    c = rng.uniform(-1, 1, (F, 1, 3))
    V = (c + rng.standard_normal((F, 3, 3)) * rng.uniform(0.001, 0.2, (F, 1, 1))).reshape(-1, 3).astype(np.float32)
    o = rng.uniform(-1.5, 1.5, (20000, 3)).astype(np.float32)
    check(V, np.arange(3 * F).reshape(-1, 3), o, rand_dirs(rng, 20000))
    # a finite window, directions of length 7.5
    check(V, np.arange(3 * F).reshape(-1, 3), o, rand_dirs(rng, 20000) * np.float32(7.5), tnear=0.05, tfar=0.3)


@pytest.mark.parametrize("name", ["sphere", "torus", "two_spheres"])
def test_marching_cubes_meshes(cuda, name):
    if name == "two_spheres":
        V, F, _ = two_spheres()
    else:
        vol = C.sphere_volume((30,) * 3, (14.3, 14.6, 14.1), 11.0) if name == "sphere" else C.torus_volume((40, 40, 20), (19.4, 19.7, 9.6),
                                                                                                              13.0, 5.0)
        V, F = mc_mesh(vol)
    rng = np.random.default_rng(3)
    lo, hi = V.min(0) - 2, V.max(0) + 2
    n = 6000
    o = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    tgt = V[rng.integers(0, V.shape[0], n)]
    check(V, F, o, (tgt - o).astype(np.float32))
    check(V, F, o, rand_dirs(rng, n))
    # origins inside the mesh (the centre region) and on the vertices themselves
    c = (V.min(0) + V.max(0)) / 2
    check(V, F, (c + rng.uniform(-1, 1, (n, 3))).astype(np.float32), rand_dirs(rng, n), expect_some=False)
    idx = rng.integers(0, V.shape[0], n)
    check(V, F, V[idx], rand_dirs(rng, n), tnear=1e-4, expect_some=False)


def test_axis_aligned_box_floor_and_ties(cuda):
    """zero-thickness boxes; axis-parallel rays (directions with zero components), origins on box planes, rays aimed at shared edges and
    vertices, where the faces on both sides pass at the same t and the smaller index must win, and grazing rays"""
    bV, bF = box_mesh((0.0, 0.0, 0.0), (1.0, 2.0, 0.5))
    gV, gF = floor_grid(8, z=-1.0)
    V = np.concatenate([bV, gV])
    F = np.concatenate([bF, gF + bV.shape[0]])
    rng = np.random.default_rng(5)
    axes = np.concatenate([np.eye(3), -np.eye(3)]).astype(np.float32)
    grid = np.arange(-2, 10) * np.float32(0.25)
    pts = np.stack(np.meshgrid(grid, grid, np.array([-1.0, -0.5, 0.0, 0.25, 0.5, 1.0], np.float32), indexing="ij"), -1).reshape(-1, 3)
    o = np.repeat(pts, 6, 0).astype(np.float32)
    d = np.tile(axes, (pts.shape[0], 1))
    check(V, F, o, d, tnear=-1e-4)
    check(V, F, o, d, tnear=1e-4)
    tgt = np.concatenate([gV, (gV[gF[:, 0]] + gV[gF[:, 1]]) / 2, bV, (bV[bF[:, 0]] + bV[bF[:, 2]]) / 2]).astype(np.float32)
    src = (tgt + rng.uniform(-3, 3, tgt.shape)).astype(np.float32)
    _, rf, _ = check(V, F, src, (tgt - src).astype(np.float32))
    # straight down onto the floor's vertices and edge midpoints: ties between the faces that share them
    down = np.tile(np.float32([0, 0, -1]), (tgt.shape[0], 1))
    _, rf, _ = check(V, F, (tgt + np.float32([0, 0, 3])).astype(np.float32), down, expect_some=False)
    assert (rf >= 0).all()
    n = 6000
    o = np.concatenate([rng.uniform(-0.5, 2.5, (n, 2)), np.full((n, 1), -1.0) + rng.choice([0.0, 1e-6, -1e-6], (n, 1))], 1).astype(np.float32)
    d = np.concatenate([rand_dirs(rng, n)[:, :2], rng.choice([0.0, 1e-3, -1e-3, 1e-7], (n, 1))], 1).astype(np.float32)
    check(V, F, o, d, tnear=-1.0)


def test_degenerate_faces_and_tiny_meshes(cuda):
    rng = np.random.default_rng(7)
    ang = np.linspace(0, 2 * np.pi, 64, endpoint=False)[:, None] + np.array([0, 2 * np.pi / 3, 4 * np.pi / 3])[None]
    tri = np.stack([np.cos(ang), np.sin(ang), np.zeros_like(ang)], -1) * 0.5
    tri[..., 2] = np.linspace(-0.1, 0.1, 64)[:, None] * np.array([1, -1, 0])[None]
    V = np.concatenate([tri.reshape(-1, 3), tri.reshape(-1, 3)]).astype(np.float32)
    F = np.concatenate([np.arange(V.shape[0]).reshape(-1, 3), [[0, 0, 1], [2, 2, 2]]])
    o = rng.uniform(-1, 1, (20000, 3)).astype(np.float32)
    d = rand_dirs(rng, 20000)
    check(V, F, o, d)
    check(np.zeros((9, 3), np.float32), np.arange(9).reshape(-1, 3), o, d, expect_some=False)
    check(V[:3], [[0, 1, 2]], o, d)
    t, f, b = check(V[:3], np.zeros((0, 3), int), o, d, expect_some=False)
    assert (f == -1).all() and np.isinf(t).all() and (b == 0).all()


@pytest.mark.parametrize("R", [1, 257, 2 ** 20 + 3])
def test_ray_counts_and_repeatability(cuda, R):
    rng = np.random.default_rng(R)
    V, F = mc_mesh(C.torus_volume((24, 24, 14), (11.4, 11.7, 6.6), 7.0, 3.0))
    o = rng.uniform(-2, 26, (R, 3)).astype(np.float32)
    d = rand_dirs(rng, R)
    if R < 2 ** 20:
        check(V, F, o, d, expect_some=R > 100)
    m = Mesh(cu(V), cu(F, torch.int32))
    a = m.first_hit(cu(o), cu(d))
    b = m.first_hit(cu(o), cu(d))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    if R > 1000:
        assert bool((a[1] >= 0).any())


# ------------------------------------------------------------------------------------------------ render == shade(first_hit(reel rays))
def reel_rays(K, tf, H, W):
    """every pixel of every image through the training ray kernel -> (o, d) [I H W, 3] in image, row, column order"""
    from permuto_sdf_b200.permuto_sdf import PermutoSDF
    I = K.shape[0]
    reel = TensorReel(torch.zeros(I, 3, H, W, device="cuda"), None, K, tf)
    pix = torch.arange(H * W, dtype=torch.int32, device="cuda").repeat(I)
    img = torch.arange(I, dtype=torch.int32, device="cuda").repeat_interleave(H * W)
    o, d, _, _, _ = PermutoSDF.rays_from_reel_indices(reel, pix, img)
    return o.cpu().numpy(), d.cpu().numpy()


def nchw(x, I, H, W):
    """[I H W, C] or [I H W] rows -> [I,C,H,W]"""
    x = x.reshape(I, H, W, -1)
    return np.ascontiguousarray(x.transpose(0, 3, 1, 2))


@pytest.mark.parametrize("with_nv,with_colors", [(False, False), (True, False), (False, True), (True, True)])
def test_render_equals_shade_of_the_reel_rays(cuda, with_nv, with_colors):
    V, F = mc_mesh(C.torus_volume((26, 26, 14), (12.4, 12.7, 6.6), 8.0, 3.5))
    V = ((V - np.float32([12.4, 12.7, 6.6])) / np.float32(30.0)).astype(np.float32) @ rotation(2).T.astype(np.float32)
    V = V.astype(np.float32)
    m = Mesh(cu(V), cu(F, torch.int32))
    if with_nv:
        m.recalculate_normals()
    rng = np.random.default_rng(11)
    colors = rng.uniform(0, 1, V.shape).astype(np.float32) if with_colors else None
    H, W, I = 24, 40, 3
    K, tf = sphere_cameras(I, H, W, 30.0, radius=1.0)
    tf[1, :3, 3] += torch.tensor([0.05, -0.02, 0.01], device="cuda")        # off-centre: rays not symmetric about the principal point
    out = m.render(K, tf, H, W, colors=None if colors is None else cu(colors))
    assert set(out) == set(RENDER_OUTPUTS)
    o, d = reel_rays(K, tf, H, W)
    ref = FH.shade(V, F, *FH.first_hit(V, F, o, d), normals=m.NV.cpu().numpy() if with_nv else None, colors=colors)
    for k in RENDER_OUTPUTS:
        got = out[k].cpu().numpy()
        want = nchw(ref[k], I, H, W)
        assert got.shape == want.shape and got.dtype == want.dtype, k
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (k, np.flatnonzero(got != want)[:10])
    hits = (out["mask"] > 0).float().mean().item()
    assert 0.05 < hits < 0.95, hits
    # any subset of outputs, the same bits; the same bits on every run
    for sub in (("depth",), ("face", "rgb"), ("normal", "mask")):
        part = m.render(K, tf, H, W, colors=None if colors is None else cu(colors), outputs=sub)
        assert set(part) == set(sub) and all(torch.equal(part[k], out[k]) for k in sub)
    again = m.render(K, tf, H, W, colors=None if colors is None else cu(colors))
    assert all(torch.equal(again[k], out[k]) for k in RENDER_OUTPUTS)


def test_render_sizes_and_window(cuda):
    """image sizes that are not multiples of the 8 x 4 warp tile, a one-pixel image, and a (tnear, tfar) window"""
    V, F = box_mesh((-0.3, -0.2, -0.25), (0.3, 0.2, 0.25))
    m = Mesh(cu(V), cu(F, torch.int32))
    for H, W in ((1, 1), (5, 13), (33, 7)):
        K, tf = sphere_cameras(2, H, W, 0.8 * max(H, W), radius=1.5)
        out = m.render(K, tf, H, W, tnear=1.2, tfar=1.6)
        o, d = reel_rays(K, tf, H, W)
        ref = FH.shade(V, F, *FH.first_hit(V, F, o, d, np.float32(1.2), np.float32(1.6)))
        for k in RENDER_OUTPUTS:
            assert np.array_equal(out[k].cpu().numpy().view(np.int32), nchw(ref[k], 2, H, W).view(np.int32)), (H, W, k)


def test_rendered_sphere_matches_the_analytic_reel(cuda):
    """a marching-cubes sphere of radius 0.3 (256^3 grid over [-0.5, 0.5]^3, normals from recalculate_normals) rendered with
    bench.analytic_reel's K and tf: the mask agrees except on pixels next to the silhouette, and on interior pixels (all 8 neighbours
    inside) the rgb agrees within 5e-3. Measured on an H100 80GB HBM3 (700 W): the largest interior rgb difference 3.5e-3."""
    import bench
    N, H, W = 256, 60, 80
    reel = bench.analytic_reel(6, H, W, 100.0, torch.device("cuda"))
    g = (torch.arange(N, device="cuda", dtype=torch.float32) / (N - 1) - 0.5)
    x, y, z = torch.meshgrid(g, g, g, indexing="ij")
    V, F = marching_cubes((torch.sqrt(x * x + y * y + z * z) - 0.3).contiguous())
    m = Mesh(V / (N - 1) - 0.5, F).recalculate_normals()
    out = m.render(reel.K_reel, reel.tf_world_cam_reel, H, W, outputs=("rgb", "mask"))
    ref = reel.mask_reel
    pool = lambda a: torch.nn.functional.max_pool2d(a, 3, 1, 1)
    edge = (pool(ref) != -pool(-ref))                     # pixels with a neighbour on the other side of the silhouette
    assert torch.equal(out["mask"][~edge], ref[~edge])
    inner = (-pool(-ref) > 0).expand(-1, 3, -1, -1)
    diff = float((out["rgb"] - reel.rgb_reel)[inner].abs().max())
    print("largest interior rgb difference %.3g" % diff)
    assert diff < 5e-3, diff


def test_refusals(cuda):
    V, F = box_mesh((0, 0, 0), (1, 1, 1))
    m = Mesh(cu(V), cu(F, torch.int32))
    K, tf = sphere_cameras(2, 8, 8, 10.0, radius=3.0)
    cases = [
        (dict(K=K[:, :2]), "K must be a tensor of shape"),
        (dict(K=K.double()), "K must be float32"),
        (dict(K=K.cpu()), "K must be on V's device"),
        (dict(tf_world_cam=tf[:1]), "1 tf_world_cam"),
        (dict(tf_world_cam=tf.clone().index_fill_(1, torch.tensor([0], device="cuda"), float("nan"))), "tf_world_cam has values that"),
        (dict(K=K.clone().fill_(float("inf"))), "K has values that are not finite"),
        (dict(H=0), "H must be a positive integer"),
        (dict(W=2.5), "W must be a positive integer"),
        (dict(H=65536, W=65536), "2\\^31"),
        (dict(colors=torch.zeros(8, 3, dtype=torch.float64, device="cuda")), "colors must be a float32 tensor"),
        (dict(colors=torch.zeros(7, 3, device="cuda")), "colors must be a float32 tensor"),
        (dict(colors=torch.zeros(8, 3)), "colors must be on V's device"),
        (dict(outputs=("rgb", "albedo")), "unknown output 'albedo'"),
        (dict(tnear=math.inf), "tnear must be finite"),
    ]
    for kw, match in cases:
        args = dict(K=K, tf_world_cam=tf, H=8, W=8)
        args.update(kw)
        with pytest.raises(RuntimeError, match=match):
            m.render(**args)
    with pytest.raises(RuntimeError, match="NV must be"):
        Mesh(m.V, m.F, torch.zeros(8, 2, device="cuda")).render(K, tf, 8, 8)
    bad = Mesh(m.V, cu(np.concatenate([F, [[0, 1, 8]]]), torch.int32))
    with pytest.raises(RuntimeError, match="outside"):
        bad.render(K, tf, 8, 8)
    with pytest.raises(RuntimeError, match="outside"):
        bad.first_hit(torch.zeros(1, 3, device="cuda"), torch.ones(1, 3, device="cuda"))
    with pytest.raises(RuntimeError, match="finite"):
        m.first_hit(torch.full((1, 3), float("nan"), device="cuda"), torch.ones(1, 3, device="cuda"))
    with pytest.raises(RuntimeError, match="shape"):
        m.first_hit(torch.zeros(1, 4, device="cuda"), torch.ones(1, 4, device="cuda"))
    with pytest.raises(RuntimeError, match="CUDA"):
        Mesh(m.V.cpu(), m.F.cpu()).render(K, tf, 8, 8)


# ------------------------------------------------------------------------------------------------ end to end
def test_a_torus_trained_from_its_renders(cuda):
    """A marching-cubes torus (R = 0.27, r = 0.1, inside radius 0.45), 24 sphere_cameras views at 96 x 128 with masks. Trainer(nr_images=24,
    deterministic=True), fit_sphere(), then STEPS = 1000 step_from_reel iterations of 512 pixels drawn from images 0-20 (seeded); 1000
    steps took 11 s, the sphere fit 22 s, the whole test 29 s. Measured on an H100 80GB HBM3 (700 W), two runs: held-out PSNR on images
    21-23 14.51 and 14.57 dB (bar 13.5), chamfer of the extracted largest component against the torus 0.0172 and 0.0168 (bar 0.025),
    Euler characteristic 0 (genus 1) in both. Longer runs of the same seed: 16.37 dB, 0.0125 at 2000 steps; 17.95 dB, 0.0118 at 4000; 21.05 dB, 0.0118 at 8000."""
    from permuto_sdf_b200 import extract_mesh_from_sdf_model, mesh_distance
    from permuto_sdf_b200.train import Trainer
    N = 160
    g = torch.arange(N, device="cuda", dtype=torch.float32) / (N - 1) - 0.5
    x, y, z = torch.meshgrid(g, g, g, indexing="ij")
    q = torch.sqrt(x * x + y * y) - 0.27
    V, F = marching_cubes((torch.sqrt(q * q + z * z) - 0.1).contiguous())
    torus = Mesh(V / (N - 1) - 0.5, F).recalculate_normals()
    H, W, I = 96, 128, 24
    K, tf = sphere_cameras(I, H, W, 112.0)
    img = torus.render(K, tf, H, W, outputs=("rgb", "mask"))
    reel = TensorReel(img["rgb"], img["mask"], K, tf)
    tr = Trainer(nr_images=I, deterministic=True)
    tr.fit_sphere()
    gen = torch.Generator().manual_seed(0)
    for _ in range(STEPS):
        pix = torch.randint(0, H * W, (512,), generator=gen, dtype=torch.int32)
        im = torch.randint(0, 21, (512,), generator=gen, dtype=torch.int32)
        tr.step_from_reel(reel, pix, im)
    psnr = tr.evaluate(reel, [21, 22, 23])["psnr_mean"]
    mesh = extract_mesh_from_sdf_model(tr.model_sdf, 256, -0.5, 0.5).keep_largest_component()
    chamfer = mesh_distance(mesh, torus, nr_samples=200_000)["chamfer"]
    euler = C.euler_characteristic(mesh.F.cpu().numpy())
    print("torus: held-out PSNR %.2f dB, chamfer %.3g, Euler characteristic %d" % (psnr, chamfer, euler))
    assert psnr >= PSNR_MIN, psnr
    assert chamfer <= CHAMFER_MAX, chamfer
    assert euler == 0, euler
