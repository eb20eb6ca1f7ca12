"""load_mesh_sequence and SpaceTimeFit.from_mesh_sequence on synthetic frames: a sphere whose centre and radius move from frame to frame
(one topology), with a small closed sphere inside it that ambient occlusion removes; OBJ and PLY files written to a temporary folder."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mesh_checks as C
from permuto_sdf_b200.mesh import Mesh, load_mesh_sequence, marching_cubes

pytestmark = pytest.mark.gpu

CENTRE0, DCENTRE = np.array([0.3, -0.2, 0.1]), np.array([0.04, 0.03, -0.02])
RADIUS0, DRADIUS = 1.0, 0.03


def unit_spheres(n):
    """outer unit sphere and inner sphere of radius 0.3, both about the origin, rotated out of the grid planes of marching cubes (a ray in
    such a plane meets rows of shared edges exactly, where the fp32 test may pass neither face) -> (V [V,3] fp64, F, outer vertex count)"""
    c = (n - 1) / 2 + 0.31
    V0, F0 = marching_cubes(torch.from_numpy(C.sphere_volume((n,) * 3, (c, c, c), (n - 3) / 2)).cuda())
    V1, F1 = marching_cubes(torch.from_numpy(C.sphere_volume((n,) * 3, (c, c, c), 0.3 * (n - 3) / 2)).cuda())
    V0, V1 = (V0.double().cpu().numpy() - c) / ((n - 3) / 2), (V1.double().cpu().numpy() - c) / ((n - 3) / 2)
    q, _ = np.linalg.qr(np.random.default_rng(11).standard_normal((3, 3)))
    return np.concatenate([V0, V1]) @ q.T, np.concatenate([F0.cpu().numpy(), F1.cpu().numpy() + V0.shape[0]]), V0.shape[0]


def write_obj(path, V, Fc):
    with open(path, "w") as f:
        f.writelines("v %.9g %.9g %.9g\n" % tuple(v) for v in V)
        f.writelines("f %d %d %d\n" % tuple(t + 1) for t in Fc)


def write_frames(folder, nframes, n=28, names=None):
    U, Fc, n_outer = unit_spheres(n)
    for i in range(nframes):
        V = (U * (RADIUS0 + i * DRADIUS) + (CENTRE0 + i * DCENTRE)).astype(np.float32)
        name = names[i] if names else "frame_%d.%s" % (i, "obj" if i % 2 == 0 else "ply")
        if name.endswith(".obj"):
            write_obj(folder / name, V, Fc)
        else:
            Mesh(torch.from_numpy(V), torch.from_numpy(Fc.astype(np.int32))).save_to_file(str(folder / name))
    return n_outer


def by_hand(folder, files):
    """the reference's steps, one Mesh operation at a time"""
    frames = []
    for i, name in enumerate(files):
        m = Mesh.load(str(folder / name))
        if i == 0:
            s = m.normalize_size()
            c = m.normalize_position()
        else:
            m.scale_mesh(s)
            m.translate(-c)
        m.recalculate_normals()
        m.upsample(2, True)
        if i == 0:
            mask = m.ambient_occlusion(100) < 0.01
        m.remove_marked_vertices(mask, False)
        m.remove_unreferenced_verts()
        frames.append(m)
    meshes = [frames[i].interpolate(frames[i + 1], j / 20).recalculate_normals() for i in range(len(frames) - 1) for j in range(20)]
    K = len(meshes)
    pts = torch.cat([torch.cat([m.V, torch.full((m.V.shape[0], 1), k / (K - 1), device="cuda")], 1) for k, m in enumerate(meshes)])
    return pts, torch.cat([m.NV for m in meshes]), frames, s, c


def test_rows_match_the_reference_order(cuda, tmp_path):
    # natural order differs from lexicographic order here: frame_10 comes last
    names = ["frame_%d.%s" % (i, "obj" if i % 2 == 0 else "ply") for i in (0, 1, 2, 10)]
    write_frames(tmp_path, 4, names=names)
    (tmp_path / "readme.txt").write_text("not a mesh")
    pts, nrm = load_mesh_sequence(tmp_path)
    ref_pts, ref_nrm, frames, _, _ = by_hand(tmp_path, names)
    assert pts.dtype == torch.float32 and pts.shape[1] == 4 and nrm.shape == (pts.shape[0], 3)
    assert torch.equal(pts, ref_pts) and torch.equal(nrm, ref_nrm)
    K, nv = 60, frames[0].V.shape[0]
    assert pts.shape[0] == K * nv
    t = pts[:, 3].view(K, nv)
    assert (t == t[:, :1]).all()
    assert t[:, 0].cpu().tolist() == [float(np.float32(k / (K - 1))) for k in range(K)]
    assert float(t[0, 0]) == 0.0 and float(t[-1, 0]) == 1.0


def test_the_inner_sphere_is_removed(cuda, tmp_path):
    n_outer = write_frames(tmp_path, 2)
    pts, _ = load_mesh_sequence(tmp_path)
    m = Mesh.load(str(tmp_path / "frame_0.obj"))
    nv_all = m.V.shape[0]
    s = m.normalize_size()
    c = m.normalize_position()
    m.recalculate_normals().upsample(2, True)
    # the outer sphere alone, subdivided the same way: its vertices are the first ones and all of them stay
    o = Mesh.load(str(tmp_path / "frame_0.obj"))
    o.remove_marked_vertices(torch.arange(nv_all, device="cuda") < n_outer, True)
    o.scale_mesh(s)
    o.translate(-c)
    o.recalculate_normals().upsample(2, True)
    K = 20
    first = pts[:pts.shape[0] // K, :3]
    assert torch.equal(first, o.V)
    assert first.shape[0] < m.V.shape[0]


def test_refusals(cuda, tmp_path):
    write_frames(tmp_path, 2)
    V, Fc, _ = unit_spheres(20)
    write_obj(tmp_path / "frame_2.obj", V.astype(np.float32), Fc)
    with pytest.raises(RuntimeError, match="frame_2.obj"):
        load_mesh_sequence(tmp_path)
    one = tmp_path / "one"
    one.mkdir()
    write_frames(one, 1)
    with pytest.raises(RuntimeError, match="at least 2"):
        load_mesh_sequence(one)


def test_convergence(cuda, tmp_path):
    from permuto_sdf_b200 import SpaceTimeFit
    nframes = 3
    write_frames(tmp_path, nframes, n=40)
    torch.manual_seed(123)
    f = SpaceTimeFit.from_mesh_sequence(tmp_path)
    m = Mesh.load(str(tmp_path / "frame_0.obj"))
    s = m.normalize_size()
    c = m.normalize_position().double().cpu().numpy()
    K = 20 * (nframes - 1)
    if f.direct:
        f.enable_cuda_graph()
    f.fit(3000)
    torch.cuda.synchronize()
    g = torch.Generator(device="cuda").manual_seed(2)
    th = ((torch.arange(200, device="cuda").double() + 0.5) / 200).repeat_interleave(50)          # held-out times
    frame = th * (K - 1) / 20                                                                         # geometry, in frames
    centre = (torch.from_numpy(CENTRE0).cuda()[None] + frame[:, None] * torch.from_numpy(DCENTRE).cuda()[None]) * s - torch.from_numpy(c).cuda()
    radius = (RADIUS0 + frame * DRADIUS) * s
    d = F.normalize(torch.randn(th.shape[0], 3, device="cuda", generator=g, dtype=torch.float64), dim=-1)
    hp = torch.cat([centre + radius[:, None] * d, th[:, None]], 1).float().contiguous()
    tb = torch.rand(200000, 1, device="cuda", generator=g, dtype=torch.float64)
    box = torch.rand(200000, 3, device="cuda", generator=g, dtype=torch.float64) - 0.5
    fb = tb[:, 0] * (K - 1) / 20
    cb = (torch.from_numpy(CENTRE0).cuda()[None] + fb[:, None] * torch.from_numpy(DCENTRE).cuda()[None]) * s - torch.from_numpy(c).cuda()
    ts = (box - cb).norm(dim=1) - (RADIUS0 + fb * DRADIUS) * s
    far = ts.abs() > 0.05
    with torch.no_grad():
        fs = f.model_sdf.fused
        sdf, grad, _ = fs(hp, f.iter_nr, with_gradient=True, with_geom=False)
        s_box, _, _ = fs(torch.cat([box, tb], 1)[far].float().contiguous(), f.iter_nr, with_gradient=False, with_geom=False)
    mean_abs = float(sdf.abs().mean())
    mean_cos = float((1 - F.cosine_similarity(grad.double(), d, dim=-1)).mean())
    sign_ok = float(((s_box.view(-1) > 0) == (ts[far] > 0)).float().mean())
    print("mesh-sequence fit: mean |sdf| %.3e, mean 1 - cos %.3e, sign correct %.5f" % (mean_abs, mean_cos, sign_ok))
    assert mean_abs < 1.5e-3 and mean_cos < 1.5e-2 and sign_ok >= 0.999, (mean_abs, mean_cos, sign_ok)
