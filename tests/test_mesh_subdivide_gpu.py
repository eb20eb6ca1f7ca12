"""Mesh subdivision on the GPU (csrc/mesh_subdivide.cu, Mesh.upsample): V and F bit-equal to oracle/subdivide.py in both modes for 1 to 3
rounds on marching-cubes meshes (a sphere, a torus, a random field cropped so that it has boundaries, and a mesh with a non-manifold
edge); the same bits on a second run; NV recalculated; bad faces refused; and remove_duplicate_vertices giving back the connectivity of
an extracted mesh from its STL export."""
import numpy as np
import pytest
import torch

import mesh_checks as C
from oracle import decimate as D
from oracle import marching_cubes as MC
from oracle import subdivide as S

pytestmark = pytest.mark.gpu


def _remove(V, F, keep):
    new_id = np.cumsum(keep) - 1
    return V[keep], new_id[F[keep[F].all(1)]]


def _cropped_random():
    V, F = MC.marching_cubes(C.random_field((30, 30, 30), seed=5), 0.0)
    return _remove(V, F, V[:, 0] < 17.3)


def _non_manifold():
    """a sphere with a fin: two extra faces on one of its edges, so that edge is in four faces and its ends in many"""
    V, F = MC.marching_cubes(C.sphere_volume((16,) * 3, (7.3, 7.6, 7.1), 5.0), 0.0)
    a, b = F[0, 0], F[0, 1]
    V = np.concatenate([V, [V[a] + [0, 0, 3.0], V[b] + [0, 3.0, 0]]]).astype(np.float32)
    n = len(V)
    return V, np.concatenate([F, [[a, b, n - 2], [b, a, n - 1]]])


MESHES = {
    "sphere": lambda: MC.marching_cubes(C.sphere_volume((24,) * 3, (11.3, 11.6, 11.1), 9.0), 0.0),
    "torus": lambda: MC.marching_cubes(C.torus_volume((32, 32, 16), (15.4, 15.7, 7.6), 10.0, 4.0), 0.0),
    "cropped_random": _cropped_random,
    "non_manifold": _non_manifold,
}


def gpu_mesh(V, F, NV=None):
    from permuto_sdf_b200.mesh import Mesh
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).cuda()
    return Mesh(t(V, np.float32), t(F, np.int32), None if NV is None else t(NV, np.float32))


def bits(t):
    return t.cpu().numpy().view(np.int32)


@pytest.mark.parametrize("rounds", [1, 2, 3])
@pytest.mark.parametrize("smooth", [False, True])
@pytest.mark.parametrize("name", sorted(MESHES))
def test_upsample_matches_oracle(cuda, name, smooth, rounds):
    V, F = MESHES[name]()
    m = gpu_mesh(V, F).upsample(rounds, smooth)
    Vo, Fo = S.upsample(V, F, rounds, smooth)
    assert m.NV is None
    assert np.array_equal(m.F.cpu().numpy(), Fo)
    assert np.array_equal(bits(m.V), Vo.view(np.int32))
    if name != "non_manifold":
        assert C.euler_characteristic(Fo) == C.euler_characteristic(F)


def test_two_runs_give_the_same_bits_and_nv_is_recalculated(cuda):
    V, F = MESHES["torus"]()
    a = gpu_mesh(V, F, np.ones_like(V)).upsample(2, True)
    b = gpu_mesh(V, F, np.ones_like(V)).upsample(2, True)
    assert torch.equal(a.V, b.V) and torch.equal(a.F, b.F)
    Vo, Fo = S.upsample(V, F, 2, True)
    assert np.array_equal(bits(a.NV), D.normals(Vo, Fo).view(np.int32)) and torch.equal(a.NV, b.NV)
    assert C.closed_and_oriented(Fo, len(Vo))


def test_vertices_without_faces_are_carried_over(cuda):
    V, F = MESHES["sphere"]()
    V = np.concatenate([V, [[100.0, 100.0, 100.0]]]).astype(np.float32)
    m = gpu_mesh(V, F).upsample(1, True)
    assert np.array_equal(m.V[len(V) - 1].cpu().numpy(), V[-1])
    assert np.array_equal(bits(m.V), S.upsample(V, F, 1, True)[0].view(np.int32))


def test_bad_faces_are_refused(cuda):
    V, F = MESHES["sphere"]()
    with pytest.raises(RuntimeError, match=r"outside \[0"):
        gpu_mesh(V, np.concatenate([F, [[0, 1, len(V)]]])).upsample(1, True)
    with pytest.raises(RuntimeError, match="repeat a vertex"):
        gpu_mesh(V, np.concatenate([F, [[0, 1, 1]]])).upsample(1, False)


def test_oversized_result_is_refused_before_any_allocation(cuda):
    from permuto_sdf_b200.mesh import Mesh
    m = Mesh(torch.zeros(3, 3, device="cuda"), torch.tensor([[0, 1, 2]], dtype=torch.int32, device="cuda").expand(2 ** 29, 3))
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(RuntimeError, match="2\\^31"):
        m.upsample(1, True)
    assert torch.cuda.memory_allocated() == before


def test_weld_of_an_stl_export_gives_back_the_connectivity(cuda, tmp_path):
    from permuto_sdf_b200.mesh import Mesh
    V, F = MC.marching_cubes(C.torus_volume((40, 40, 20), (19.4, 19.7, 9.6), 12.0, 5.0), 0.0)
    rec = np.zeros(len(F), dtype=[("n", "<f4", (3,)), ("v", "<f4", (3, 3)), ("attr", "<u2")])
    rec["v"] = V[F]
    p = tmp_path / "t.stl"
    p.write_bytes(b"solid torus".ljust(80, b" ") + np.uint32(len(F)).tobytes() + rec.tobytes())
    m = Mesh.load(str(p))
    assert m.V.is_cuda and m.NV is None
    # first-occurrence renumbering of the original vertices
    order = np.unique(F.reshape(-1), return_index=True)
    first = np.argsort(order[1])
    new_of_old = np.empty(len(V), np.int64)
    new_of_old[order[0][first]] = np.arange(len(first))
    assert np.array_equal(m.F.cpu().numpy(), new_of_old[F])
    assert np.array_equal(m.V.cpu().numpy(), V[order[0][first]])
