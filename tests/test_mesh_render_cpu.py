"""The first-hit oracle (tests/first_hit_oracle.py: first_hit, shade) against an fp64 intersection on simple scenes, the tie rule on coincident
faces, the camera conventions of cameras.py (look_at gives bench.analytic_reel's tf bit for bit) and TensorReel's refusals. No GPU."""
import math

import numpy as np
import pytest
import torch

import bench
import first_hit_oracle as FH
from permuto_sdf_b200.cameras import TensorReel, look_at, orbit_cameras, sphere_cameras
from permuto_sdf_b200.mesh import fibonacci_directions


def first_hit_fp64(V, F, o, d, tnear=0.0, tfar=math.inf):
    """Moller-Trumbore in fp64 over every face -> (t [R], face [R]): the smallest t, ties to the smallest face"""
    V, F = np.asarray(V, np.float64), np.asarray(F, np.int64).reshape(-1, 3)
    o, d = np.asarray(o, np.float64)[:, None], np.asarray(d, np.float64)[:, None]
    p0, p1, p2 = V[F[:, 0]][None], V[F[:, 1]][None], V[F[:, 2]][None]
    e1, e2 = p1 - p0, p2 - p0
    pv = np.cross(d, e2)
    det = (e1 * pv).sum(-1)
    with np.errstate(all="ignore"):
        tv = o - p0
        u = (tv * pv).sum(-1) / det
        qv = np.cross(tv, e1)
        v = (d * qv).sum(-1) / det
        t = (e2 * qv).sum(-1) / det
    ok = (det != 0) & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (t > tnear) & (t < tfar)
    t = np.where(ok, t, np.inf)
    return t.min(1), np.where(ok.any(1), np.argmin(t, 1), -1)


def box_mesh(lo, hi):
    x = np.array([[lo[0], lo[1], lo[2]], [hi[0], lo[1], lo[2]], [hi[0], hi[1], lo[2]], [lo[0], hi[1], lo[2]],
                  [lo[0], lo[1], hi[2]], [hi[0], lo[1], hi[2]], [hi[0], hi[1], hi[2]], [lo[0], hi[1], hi[2]]], np.float32)
    F = np.array([[0, 2, 1], [0, 3, 2], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4], [2, 3, 7], [2, 7, 6], [1, 2, 6], [1, 6, 5],
                  [0, 4, 7], [0, 7, 3]])
    return x, F


def floor_grid(n, h=0.25, z=0.0):
    x, y = np.meshgrid(np.arange(n + 1) * h, np.arange(n + 1) * h, indexing="ij")
    V = np.stack([x.ravel(), y.ravel(), np.full(x.size, z)], 1).astype(np.float32)
    i = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]).ravel()
    return V, np.concatenate([np.stack([i, i + n + 1, i + 1], 1), np.stack([i + 1, i + n + 1, i + n + 2], 1)])


def rand_dirs(rng, n):
    d = rng.standard_normal((n, 3))
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def agree(V, F, o, d, tnear=0.0, tfar=math.inf):
    """first_hit_oracle.first_hit against fp64: the same face wherever fp64 sees no other face within 1e-4 of the first t (and the ray keeps 1e-3
    away from edges, where fp32 and fp64 may pick different neighbours), t within 1e-5 relative, bary consistent with the hit point"""
    t, f, b = FH.first_hit(V, F, o, d, tnear, tfar)
    t64, f64 = first_hit_fp64(V, F, o, d, tnear, tfar)
    assert t.dtype == np.float32 and f.dtype == np.int32 and b.dtype == np.float32 and b.shape == (len(o), 3)
    miss = f < 0
    assert np.array_equal(miss, f64 < 0)
    assert np.isinf(t[miss]).all() and (b[miss] == 0).all()
    h = ~miss
    assert np.allclose(t[h], t64[h], rtol=1e-5, atol=1e-6)
    Vf, Fi = np.asarray(V, np.float64), np.asarray(F, np.int64).reshape(-1, 3)
    tri = Vf[Fi[f[h]]]
    p = (b[h, :1] * tri[:, 0] + b[h, 1:2] * tri[:, 1]) + b[h, 2:3] * tri[:, 2]
    assert np.allclose(p, o[h] + t[h, None].astype(np.float64) * d[h], atol=1e-5)
    assert np.allclose(b[h].sum(1), 1, atol=1e-6) and (b[h] >= -1e-7).all()
    return t, f, b, f64


def test_box_from_outside_and_inside():
    V, F = box_mesh((-0.5, -0.25, -0.75), (0.5, 0.75, 0.25))
    rng = np.random.default_rng(0)
    o = rng.uniform(-2, 2, (3000, 3)).astype(np.float32)
    tgt = rng.uniform(-0.8, 0.8, (3000, 3)) + np.float32([0, 0.25, -0.25])
    d = (tgt - o).astype(np.float32)
    t, f, _, f64 = agree(V, F, o, d)
    assert 0.2 < (f >= 0).mean() < 0.9
    # from inside, every ray hits, and the box face it hits lies on the side the ray leaves through
    oi = rng.uniform(-0.4, 0.2, (2000, 3)).astype(np.float32) + np.float32([0, 0.2, -0.2])
    di = rand_dirs(rng, 2000)
    t, f, _, _ = agree(V, F, oi, di)
    assert (f >= 0).all()


def test_floor_grid_from_above_and_a_window():
    V, F = floor_grid(8, z=-1.0)
    rng = np.random.default_rng(1)
    o = np.concatenate([rng.uniform(0.01, 1.99, (2000, 2)), rng.uniform(0.5, 2, (2000, 1))], 1).astype(np.float32)
    d = np.concatenate([rng.uniform(-0.3, 0.3, (2000, 2)), -np.ones((2000, 1))], 1).astype(np.float32)
    t, f, _, _ = agree(V, F, o, d)
    # a window that ends before the floor misses everything, one that starts after it too
    assert (FH.first_hit(V, F, o, d, 0.0, 0.1)[1] == -1).all()
    assert (FH.first_hit(V, F, o, d, 100.0)[1] == -1).all()


def test_stacked_parallel_quads_give_the_nearest():
    """ten unit quads at z = 0, 0.1, .., 0.9, faces of the far quads first: a ray up the z axis from below hits z = 0, one from above
    z = 0.9, and one started between layers the next layer along its direction"""
    quads = []
    for k in range(10)[::-1]:
        z = 0.1 * k
        quads.append(np.array([[0, 0, z], [1, 0, z], [1, 1, z], [0, 1, z]], np.float32))
    V = np.concatenate(quads)
    F = np.concatenate([np.array([[0, 1, 2], [0, 2, 3]]) + 4 * k for k in range(10)])
    rng = np.random.default_rng(2)
    n = 1000
    xy = rng.uniform(0.05, 0.95, (n, 2))
    for z0, dz, expect_z in ((-1.0, 1.0, 0.0), (2.0, -1.0, 0.9), (0.45, 1.0, 0.5), (0.45, -1.0, 0.4)):
        o = np.concatenate([xy, np.full((n, 1), z0)], 1).astype(np.float32)
        d = np.tile(np.float32([0.0, 0.0, dz]), (n, 1))
        t, f, b, _ = agree(V, F, o, d)
        hit_z = (o[:, 2] + t * d[:, 2]).astype(np.float64)
        assert np.allclose(hit_z, expect_z, atol=1e-6), (z0, dz)
        assert (f >= 0).all() and np.allclose(V[F[f][:, 0], 2], expect_z)


def test_coincident_duplicates_tie_to_the_smallest_face():
    """the same triangle three times (faces 2, 5 and 6) and once with its corners rotated (face 4), in front of a copy 5 further along z
    (faces 0, 1 and 3): the copies that share a corner order compute the same t, and the smallest of them, face 2, wins; the rotated
    copy computes t with other roundings and wins only where its t is strictly smaller"""
    tri = np.array([[0.1, 0.2, 0.0], [0.9, 0.1, 0.05], [0.4, 0.9, -0.05]], np.float32)
    other = tri + np.float32([0, 0, 5])
    V = np.concatenate([other, tri])
    A, B = [3, 4, 5], [0, 1, 2]
    F = np.array([B, B, A, B, [4, 5, 3], A, A])
    rng = np.random.default_rng(3)
    n = 2000
    o = np.concatenate([rng.uniform(0, 1, (n, 2)), np.full((n, 1), -2.0)], 1).astype(np.float32)
    d = np.concatenate([rng.uniform(-0.05, 0.05, (n, 2)), np.ones((n, 1))], 1).astype(np.float32)
    t, f, b = FH.first_hit(V, F, o, d)
    h = f >= 0
    assert h.mean() > 0.2
    ok, tt, _, _ = FH.intersect(V[F[:, 0]][None], V[F[:, 1]][None], V[F[:, 2]][None], o[:, None], d[:, None], 0.0, math.inf)
    tt = np.where(ok, tt, np.inf)
    assert np.array_equal(t[h], tt[h].min(1))
    assert np.array_equal(f[h], np.argmax(ok[h] & (tt[h] == t[h, None]), 1))
    near = h & (t < 4)
    assert near.mean() > 0.2 and set(np.unique(f[near]).tolist()) <= {2, 4}
    assert (f[near] == 2).mean() > 0.5
    # the first copy in order wins ties: face 2 whenever it hits at the smallest t
    assert (f[h & (tt[:, 2] == t)] == 2).all()


def test_degenerate_faces_and_no_faces():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0]], np.float32)
    o = np.float32([[0.2, 0.2, -1.0], [0.5, 0.0, -1.0]])
    d = np.float32([[0, 0, 1], [0, 0, 1]])
    t, f, b = FH.first_hit(V, np.zeros((0, 3), int), o, d)
    assert (f == -1).all() and np.isinf(t).all() and (b == 0).all()
    # a repeated vertex and collinear corners are never hit
    t, f, b = FH.first_hit(V, [[0, 0, 1], [0, 1, 3]], o, d)
    assert (f == -1).all()
    t, f, b = FH.first_hit(V, [[0, 0, 1], [0, 1, 2]], o, d)
    assert f.tolist()[0] == 1 and t[0] == 1


def test_shade_formulas():
    V = np.array([[0, 0, 0], [2, 0, 0], [0, 2, 0]], np.float32)
    F = [[0, 1, 2]]
    t, f, b = FH.first_hit(V, F, np.float32([[0.5, 0.5, 1.0], [5, 5, 1]]), np.float32([[0, 0, -1], [0, 0, -1]]))
    s = FH.shade(V, F, t, f, b)
    assert s["normal"][0].tolist() == [0, 0, 1] and s["rgb"][0].tolist() == [0.5, 0.5, 1.0]
    assert s["mask"].tolist() == [1, 0] and s["depth"].tolist() == [1, 0] and s["face"].tolist() == [0, -1]
    assert (s["rgb"][1] == 0).all() and (s["normal"][1] == 0).all()
    C = np.float32([[1, 0, 0], [0, 1, 0], [0, 0, 1]])
    s = FH.shade(V, F, t, f, b, colors=C)
    assert np.allclose(s["rgb"][0], [0.5, 0.25, 0.25]) and s["rgb"][0].dtype == np.float32
    # zero interpolated normals stay zero
    s = FH.shade(V, F, t, f, b, normals=np.zeros((3, 3), np.float32))
    assert (s["normal"] == 0).all() and (s["rgb"][0] == 0.5).all()


# ------------------------------------------------------------------------------------------------ cameras
def test_look_at_gives_the_analytic_reels_tf():
    reel = bench.analytic_reel(16, 12, 16, 20.0, torch.device("cpu"))
    tf = look_at(reel.tf_world_cam_reel[:, :3, 3])
    assert tf.dtype == torch.float32 and torch.equal(tf, reel.tf_world_cam_reel)


def test_look_at_conventions_and_refusals():
    eyes = torch.tensor([[0.0, 0.0, 2.0], [3.0, 1.0, -1.0]])
    tf = look_at(eyes, target=(0.0, 0.5, 0.0))
    R = tf[:, :3, :3]
    assert torch.allclose(R.transpose(1, 2) @ R, torch.eye(3).expand(2, 3, 3), atol=1e-6)
    assert torch.allclose(torch.linalg.det(R), torch.ones(2))
    z = torch.tensor([0.0, 0.5, 0.0]) - eyes
    assert torch.allclose(R[:, :, 2], z / z.norm(dim=1, keepdim=True))
    assert R[:, 1, 0].abs().max() < 1e-7, "x is horizontal"
    assert (R[:, 1, 1] > 0).all(), "y points up"
    assert torch.equal(tf[:, :3, 3], eyes) and tf[:, 3].tolist() == [[0, 0, 0, 1]] * 2
    with pytest.raises(RuntimeError, match="along up"):
        look_at(torch.tensor([[0.0, 2.0, 0.0]]))
    with pytest.raises(RuntimeError, match="at the target"):
        look_at(torch.tensor([[1.0, 2.0, 3.0]]), target=(1.0, 2.0, 3.0))
    with pytest.raises(RuntimeError, match="shape"):
        look_at(torch.zeros(2, 4))


def test_sphere_and_orbit_cameras():
    K, tf = sphere_cameras(24, 96, 128, 120.0, device="cpu")
    assert K.shape == (24, 3, 3) and tf.shape == (24, 4, 4) and K.dtype == tf.dtype == torch.float32
    assert K[5].tolist() == [[120, 0, 64], [0, 120, 48], [0, 0, 1]]
    eyes = torch.from_numpy(fibonacci_directions(24)) * 1.2
    assert torch.equal(tf[:, :3, 3], eyes) and torch.equal(tf, look_at(eyes))
    K, tf = orbit_cameras(8, 60, 80, 100.0, device="cpu")
    e = tf[:, :3, 3].double()
    assert torch.allclose(e.norm(dim=1), torch.full((8,), 1.8, dtype=torch.float64), atol=1e-6)
    assert torch.allclose(e[:, 1], torch.full((8,), 0.9, dtype=torch.float64), atol=1e-6)
    assert torch.allclose(e[0], torch.tensor([0.0, 0.9, 1.8 * math.cos(math.radians(30))], dtype=torch.float64), atol=1e-6)
    az = torch.atan2(e[:, 0], e[:, 2]) % (2 * math.pi)
    assert torch.allclose(az, torch.arange(8, dtype=torch.float64) * (math.pi / 4), atol=1e-6)
    with pytest.raises(RuntimeError, match="nr_images"):
        sphere_cameras(0, 10, 10, 10.0, device="cpu")
    with pytest.raises(RuntimeError, match="focal"):
        orbit_cameras(4, 10, 10, -1.0, device="cpu")


# ------------------------------------------------------------------------------------------------ TensorReel
def test_tensor_reel_accepts_a_reel_and_refuses_bad_ones():
    I, H, W = 3, 6, 8
    rgb, mask = torch.zeros(I, 3, H, W), torch.zeros(I, 1, H, W)
    K, tf = torch.eye(3).repeat(I, 1, 1), torch.eye(4).repeat(I, 1, 1)
    r = TensorReel(rgb, mask, K, tf)
    assert r.rgb_reel is rgb and r.mask_reel is mask and r.K_reel is K and r.tf_world_cam_reel is tf
    assert TensorReel(rgb, None, K, tf).mask_reel is None
    cases = [
        ((rgb[:, :2], mask, K, tf), "rgb must be a tensor of shape"),
        ((rgb.numpy(), mask, K, tf), "rgb must be a tensor of shape"),
        ((rgb, mask[:2], K, tf), r"mask must be a tensor of shape \[3, 1, 6, 8\]"),
        ((rgb, mask, K[:, :2], tf), "K must be a tensor of shape"),
        ((rgb, mask, K, tf[:2]), "tf_world_cam must be a tensor of shape"),
        ((rgb.double(), mask, K, tf), "rgb must be float32"),
        ((rgb, mask.half(), K, tf), "mask must be float32"),
        ((rgb, mask, K, tf.double()), "tf_world_cam must be float32"),
        ((rgb, mask, K.transpose(1, 2), tf), "K must be contiguous"),
        ((rgb, torch.zeros(I, 1, W, H).transpose(2, 3), K, tf), "mask must be contiguous"),
        ((torch.zeros(0, 3, H, W), None, K[:0], tf[:0]), "at least one image"),
    ]
    for args, match in cases:
        with pytest.raises(RuntimeError, match=match):
            TensorReel(*args)
    if torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="device"):
            TensorReel(rgb, mask, K.cuda(), tf)


# ------------------------------------------------------------------------------------------------ compile check
def test_first_hit_kernels_are_built_and_do_not_spill():
    import os
    import shutil
    import sys
    if not os.path.exists(shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"):
        pytest.skip("nvcc not available")
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import wgmma_report
    fh = {r["kernel"]: r for r in wgmma_report.report(("mesh_raycast.cu",)) if r["kernel"].startswith("k_fh_")}
    assert set(fh) == {"k_fh_rays", "k_fh_render<true>"}
    spilling = {k: (r["spill_st"], r["spill_ld"]) for k, r in fh.items() if r["spill_st"] or r["spill_ld"]}
    assert not spilling, spilling
