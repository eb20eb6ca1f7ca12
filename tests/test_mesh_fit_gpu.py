"""From a mesh file to a fitted SDF: the analytic sphere and torus of test_surface_fit_gpu.py, extracted with marching_cubes and written as
binary STL, go through the preprocessing of train_sdf_from_mesh.py:80-93 (load, weld, normalize_size, normalize_position, scale_mesh(0.6),
remove_unreferenced_verts, recalculate_normals) and one round of Loop subdivision into SurfaceFit.from_mesh(...).fit(3000). The fit is
checked against the true SDF mapped into the normalised frame through the returned scale and centre, with the metrics and thresholds of
test_convergence_on_analytic_clouds: mean |sdf| on the surface, normal cosine, and the sign off the surface."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_surface_fit_gpu import sphere_cloud, sphere_sdf, torus_cloud, torus_sdf

pytestmark = pytest.mark.gpu

N = 160                       # grid points per axis on [-0.5, 0.5]


def write_stl(path, V, Fc):
    rec = np.zeros(len(Fc), dtype=[("n", "<f4", (3,)), ("v", "<f4", (3, 3)), ("attr", "<u2")])
    rec["v"] = V[Fc]
    with open(path, "wb") as f:
        f.write(b"binary STL written by a test".ljust(80, b" ") + np.uint32(len(Fc)).tobytes() + rec.tobytes())


def test_surface_fit_from_a_mesh_in_the_constructor_checks(cuda):
    from permuto_sdf_b200 import SurfaceFit
    from permuto_sdf_b200.mesh import Mesh
    m = Mesh(torch.zeros(3, 3, device="cuda"), torch.tensor([[0, 1, 2]], dtype=torch.int32, device="cuda"))
    with pytest.raises(RuntimeError, match="no vertex normals"):
        SurfaceFit.from_mesh(m)


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_fit_from_an_stl_file(cuda, tmp_path, shape):
    from permuto_sdf_b200 import SurfaceFit
    from permuto_sdf_b200.mesh import Mesh, marching_cubes
    cloud, true_sdf = (sphere_cloud, sphere_sdf) if shape == "sphere" else (torus_cloud, torus_sdf)
    lin = torch.linspace(-0.5, 0.5, N, device="cuda")
    grid = torch.stack(torch.meshgrid(lin, lin, lin, indexing="ij"), -1).reshape(-1, 3)
    V, Fc = marching_cubes(true_sdf(grid).reshape(N, N, N).contiguous(), 0.0)       # index space: world = -0.5 + p h
    h = 1.0 / (N - 1)
    path = str(tmp_path / (shape + ".stl"))
    write_stl(path, V.cpu().numpy(), Fc.cpu().numpy())

    # the preprocessing lines of train_sdf_from_mesh.py, minus its rotations
    mesh = Mesh.load(path)
    s = mesh.normalize_size()
    c = mesh.normalize_position()
    mesh.scale_mesh(0.6)
    mesh.remove_unreferenced_verts()
    mesh.recalculate_normals()
    mesh.upsample(1, True)
    assert mesh.V.shape[0] > 4 * V.shape[0] - 10 and mesh.F.shape[0] == 4 * Fc.shape[0]
    f = SurfaceFit.from_mesh(mesh)
    f.enable_cuda_graph()
    f.fit(3000)
    torch.cuda.synchronize()

    # q (normalised) = (p s - c) 0.6 with p in index space; world = -0.5 + p h; sdf scales by s 0.6 / h
    to_world = lambda q: -0.5 + ((q / 0.6 + c) / s) * h
    to_q = lambda w: ((w + 0.5) / h * s - c) * 0.6
    k = s * 0.6 / h
    hp, hn = cloud(10000, seed=2)
    with torch.no_grad():
        sdf, grad, _ = f.model_sdf.fused(to_q(hp).contiguous(), f.iter_nr, with_gradient=True, with_geom=False)
        mean_abs = float(sdf.abs().mean())
        mean_cos = float((1 - F.cosine_similarity(grad, hn, dim=-1)).mean())
        g = torch.Generator(device="cuda").manual_seed(3)
        box = torch.rand(200000, 3, device="cuda", generator=g) - 0.5
        ts = true_sdf(to_world(box)) * k
        far = ts.abs() > 0.05
        s_box, _, _ = f.model_sdf.fused(box[far].contiguous(), f.iter_nr, with_gradient=False, with_geom=False)
        sign_ok = float(((s_box.view(-1) > 0) == (ts[far] > 0)).float().mean())
    print("mesh fit %s: %d vertices, scale %.6f, centre %s, mean |sdf| %.3e, mean 1 - cos %.3e, sign correct %.5f, loss %.4e" % (
        shape, mesh.V.shape[0], s, c.tolist(), mean_abs, mean_cos, sign_ok, float(f.last["terms"][0])))
    assert mean_abs < 2e-3 and mean_cos < 1e-2 and sign_ok >= 0.99, (mean_abs, mean_cos, sign_ok)
