"""Connected components of a mesh on the GPU (csrc/mesh_components.cu, Mesh.connected_components / remove_small_components /
keep_largest_component): the partition, the component count and the face counts against scipy.sparse.csgraph on marching-cubes meshes of
random volumes and on small hand-made meshes; a long triangle strip (the deepest union-find chains) in three vertex numberings; labels the
same bits for any face order and on every run; removal the same bits as remove_marked_vertices with a mask from scipy's components,
including a tie for the largest component; refusal of out-of-range indices; and the largest component of a mesh extracted from a
SurfaceFit of two separated spheres."""
import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph
import torch

import mesh_checks as C

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _reduction_mode_off_after(cuda):
    """SurfaceFit switches the device's reduction mode; later tests start from the default"""
    yield
    from permuto_sdf_b200 import call
    call("psdf_set_deterministic", 0, 0, 0)


def host_components(nv, F):
    """scipy's components of the vertex graph -> (labels = smallest vertex index of the component [nv] int64, count, face counts [nv]
    indexed by label, the component of each face's first vertex)"""
    F = np.asarray(F, dtype=np.int64).reshape(-1, 3)
    rows = np.concatenate([F[:, 0], F[:, 1], F[:, 2]])
    cols = np.concatenate([F[:, 1], F[:, 2], F[:, 0]])
    A = scipy.sparse.coo_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(nv, nv)).tocsr()
    n, lab = scipy.sparse.csgraph.connected_components(A, directed=False)
    smallest = np.full(n, nv, dtype=np.int64)
    np.minimum.at(smallest, lab, np.arange(nv))
    labels = smallest[lab]
    counts = np.bincount(labels[F[:, 0]], minlength=nv) if len(F) else np.zeros(nv, np.int64)
    return labels, n, counts


def mesh_of(V, F, normals=True):
    from permuto_sdf_b200.mesh import Mesh
    V = torch.as_tensor(V, dtype=torch.float32).reshape(-1, 3).cuda()
    F = (F if isinstance(F, torch.Tensor) else torch.from_numpy(np.asarray(F))).to(torch.int32).reshape(-1, 3).cuda()
    NV = torch.randn(V.shape, generator=torch.Generator().manual_seed(V.shape[0])).cuda() if normals else None
    return Mesh(V, F, NV)


def check_against_scipy(m):
    labels, nr, counts = m.connected_components(with_face_counts=True)
    ref_labels, ref_nr, ref_counts = host_components(m.V.shape[0], m.F.cpu().numpy())
    assert labels.dtype == torch.int32 and labels.shape == (m.V.shape[0],) and labels.is_cuda
    assert nr == ref_nr
    assert np.array_equal(labels.cpu().numpy(), ref_labels)
    assert np.array_equal(counts.cpu().numpy(), ref_counts)
    return ref_nr


# ------------------------------------------------------------------------------------------------ partitions against scipy
def random_volume(n, seed, sigma):
    from scipy.ndimage import gaussian_filter
    f = np.random.default_rng(seed).standard_normal((n, n, n))
    if sigma:
        f = gaussian_filter(f, sigma)
    return (f / f.std()).astype(np.float32)


# (size, smoothing, threshold): inside is value < threshold, so a low threshold gives many small blobs and 0 one connected maze
VOLUMES = [(2, 0, 0.0), (2, 0, -0.3), (17, 1.0, -1.2), (17, 1.0, 0.0), (64, 1.5, -2.0), (64, 1.5, -1.0), (64, 1.5, 0.0),
           (256, 2.0, -2.5), (256, 2.0, -1.5), (256, 2.0, 0.3)]


@pytest.mark.parametrize("size,sigma,thr", VOLUMES)
def test_marching_cubes_meshes_match_scipy(size, sigma, thr):
    from permuto_sdf_b200 import marching_cubes
    vol = random_volume(size, seed=1000 * size + int(round(10 * (thr + 5))), sigma=sigma)
    V, F = marching_cubes(torch.from_numpy(vol).cuda(), thr)
    nr = check_against_scipy(mesh_of(V, F))
    print("%d^3 at %g: %d vertices, %d faces, %d components" % (size, thr, V.shape[0], F.shape[0], nr))
    if size == 256 and thr == -2.5:
        assert nr > 1000


def test_single_triangle():
    m = mesh_of(np.eye(3), [[0, 1, 2]])
    labels, nr, counts = m.connected_components(with_face_counts=True)
    assert nr == 1 and labels.tolist() == [0, 0, 0] and counts.tolist() == [1, 0, 0]
    check_against_scipy(mesh_of(np.eye(3), [[2, 0, 1]]))


def test_vertices_no_face_references():
    m = mesh_of(np.zeros((10, 3)), [[7, 5, 2], [8, 2, 7], [9, 9, 9]])
    labels, nr, counts = m.connected_components(with_face_counts=True)
    assert labels.tolist() == [0, 1, 2, 3, 4, 2, 6, 2, 2, 9] and nr == 7
    assert counts.tolist() == [0, 0, 2, 0, 0, 0, 0, 0, 0, 1]
    check_against_scipy(m)


@pytest.mark.parametrize("nv", [0, 1, 4])
def test_mesh_without_faces(nv):
    m = mesh_of(np.zeros((nv, 3)), np.zeros((0, 3)))
    labels, nr, counts = m.connected_components(with_face_counts=True)
    assert nr == nv and labels.tolist() == list(range(nv)) and counts.tolist() == [0] * nv
    check_against_scipy(m)


# ------------------------------------------------------------------------------------------------ worst case for union-find depth
@pytest.mark.parametrize("numbering", ["along", "reversed", "random"])
def test_long_triangle_strip_is_one_component(numbering):
    nf = (1 << 22) + 3
    nv = nf + 2
    i = torch.arange(nf, device="cuda", dtype=torch.int64)
    F = torch.stack([i, i + 1, i + 2], 1)
    if numbering == "reversed":
        F = nv - 1 - F
    elif numbering == "random":
        perm = torch.randperm(nv, generator=torch.Generator().manual_seed(3)).cuda()
        F = perm[F]
    m = mesh_of(torch.zeros(nv, 3), F.int(), normals=False)
    labels, nr, counts = m.connected_components(with_face_counts=True)
    assert nr == 1
    assert int(labels.max()) == 0 and int(labels.min()) == 0
    assert int(counts[0]) == nf and int(counts[1:].abs().sum()) == 0


# ------------------------------------------------------------------------------------------------ determinism
def test_labels_do_not_depend_on_face_order_or_run():
    from permuto_sdf_b200 import marching_cubes
    V, F = marching_cubes(torch.from_numpy(random_volume(128, seed=9, sigma=1.5)).cuda(), -1.6)
    m = mesh_of(V, F)
    first, nr, counts = m.connected_components(with_face_counts=True)
    assert nr > 100
    again = m.connected_components(with_face_counts=True)
    assert torch.equal(again[0], first) and again[1] == nr and torch.equal(again[2], counts)
    g = torch.Generator().manual_seed(1)
    for _ in range(3):
        rows = torch.randperm(F.shape[0], generator=g).cuda()
        shuffled = mesh_of(V, F[rows])
        lab, n, _ = shuffled.connected_components(with_face_counts=True)
        assert torch.equal(lab, first) and n == nr
    # rotating the vertices within each face changes which vertex a face counts by, not the component
    lab, n, cnt = mesh_of(V, F[:, [1, 2, 0]]).connected_components(with_face_counts=True)
    assert torch.equal(lab, first) and n == nr and torch.equal(cnt, counts)


# ------------------------------------------------------------------------------------------------ removal against a host restatement
def same_mesh(a, b):
    return torch.equal(a.V.view(torch.int32), b.V.view(torch.int32)) and torch.equal(a.F, b.F) and a.F.dtype == torch.int32 and \
        torch.equal(a.NV.view(torch.int32), b.NV.view(torch.int32))


def clone(m):
    from permuto_sdf_b200.mesh import Mesh
    return Mesh(m.V.clone(), m.F.clone(), m.NV.clone())


@pytest.fixture(scope="module")
def blobs(cuda):
    """many components of very different sizes, plus three vertices no face references"""
    from permuto_sdf_b200 import marching_cubes
    V, F = marching_cubes(torch.from_numpy(random_volume(96, seed=5, sigma=1.5)).cuda(), -1.4)
    V = torch.cat([V, torch.rand(3, 3, device="cuda")])
    return mesh_of(V, F)


def test_remove_small_components_matches_host_mask(blobs):
    labels, nr, counts = host_components(blobs.V.shape[0], blobs.F.cpu().numpy())
    assert nr > 50 and (counts[counts > 0].min() < 20) and counts.max() > 1000
    for k in (0, 1, 2, 8, 50, int(np.median(counts[counts > 0])), int(counts.max()), int(counts.max()) + 1, 2 ** 40):
        got = clone(blobs).remove_small_components(k)
        ref = clone(blobs).remove_marked_vertices(counts[labels] >= k, True)
        assert same_mesh(got, ref), k
        if k == 0:
            assert same_mesh(got, blobs)
        if k > counts.max():
            assert got.V.shape == (0, 3) and got.F.shape == (0, 3) and got.NV.shape == (0, 3)
    assert clone(blobs).remove_small_components(np.int64(3)).F.shape[0] > 0


def test_keep_largest_component_matches_host_mask(blobs):
    labels, _, counts = host_components(blobs.V.shape[0], blobs.F.cpu().numpy())
    best = int(np.flatnonzero(counts == counts.max()).min())
    got = clone(blobs).keep_largest_component()
    ref = clone(blobs).remove_marked_vertices(labels == best, True)
    assert same_mesh(got, ref)
    assert got.connected_components()[1] == 1


def test_keep_largest_component_tie_goes_to_the_smaller_label(blobs):
    """two copies of one component; the copy listed first in F has the larger vertex ids, so face order would pick it"""
    from permuto_sdf_b200.mesh import Mesh
    one = clone(blobs).keep_largest_component()
    n, nf = one.V.shape[0], one.F.shape[0]
    V = torch.cat([one.V, one.V + 2.0])
    F = torch.cat([one.F + n, one.F])
    tie = Mesh(V, F, torch.cat([one.NV, -one.NV]))
    labels, nr, counts = tie.connected_components(with_face_counts=True)
    assert nr == 2 and int(counts[0]) == int(counts[n]) == nf
    got = clone(tie).keep_largest_component()
    assert torch.equal(got.V, one.V) and torch.equal(got.F, one.F) and torch.equal(got.NV, one.NV)
    lab = host_components(2 * n, F.cpu().numpy())[0]
    assert same_mesh(got, clone(tie).remove_marked_vertices(lab == 0, True))


def test_keep_largest_of_meshes_without_faces():
    empty = mesh_of(np.zeros((0, 3)), np.zeros((0, 3))).keep_largest_component()
    assert empty.V.shape == (0, 3) and empty.F.shape == (0, 3)
    assert mesh_of(np.zeros((0, 3)), np.zeros((0, 3))).remove_small_components(0).V.shape == (0, 3)
    # no faces: every vertex is a component of 0 faces, and the smallest label wins
    m = mesh_of(np.arange(12).reshape(4, 3), np.zeros((0, 3)))
    V0 = m.V.clone()
    assert torch.equal(m.keep_largest_component().V, V0[:1])


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("faces", [[[0, 1, 4]], [[0, -1, 2]], [[0, 1, 2], [3, 2, 2 ** 31 - 1]]])
def test_out_of_range_indices_are_refused(faces):
    m = mesh_of(np.zeros((4, 3)), faces)
    F0 = m.F.clone()
    for fn in (m.connected_components, lambda: m.remove_small_components(0), m.keep_largest_component):
        with pytest.raises(RuntimeError, match=r"outside \[0, 4\)"):
            fn()
    assert torch.equal(m.F, F0) and m.V.shape == (4, 3)


def test_faces_on_another_device_than_vertices_are_refused():
    from permuto_sdf_b200.mesh import Mesh
    with pytest.raises(RuntimeError, match="device"):
        Mesh(torch.zeros(3, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32, device="cuda")).connected_components()


def test_non_contiguous_faces():
    F = torch.tensor([[0, 1, 2, 9], [2, 3, 4, 9]], dtype=torch.int32, device="cuda")[:, :3]
    labels, nr = mesh_of(np.zeros((6, 3)), F).connected_components()
    assert labels.tolist() == [0, 0, 0, 0, 0, 5] and nr == 2


# ------------------------------------------------------------------------------------------------ an extracted mesh
BIG, SMALL = ((-0.15, 0.02, 0.0), 0.2), ((0.27, -0.03, 0.05), 0.1)


def two_sphere_cloud(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    nb = n * 4 // 5                       # about proportional to the areas (4 : 1)
    pts, nrm = [], []
    for (c, r), k in ((BIG, nb), (SMALL, n - nb)):
        d = torch.nn.functional.normalize(torch.randn(k, 3, device="cuda", generator=g), dim=-1)
        pts.append(torch.tensor(c, device="cuda") + r * d)
        nrm.append(d)
    return torch.cat(pts).contiguous(), torch.cat(nrm).contiguous()


def test_largest_component_of_an_extracted_mesh():
    from permuto_sdf_b200 import SurfaceFit, extract_mesh_from_sdf_model
    pts, nrm = two_sphere_cloud(200000)
    f = SurfaceFit(pts, nrm, nr_iters_for_c2f=500)
    assert f.direct
    f.enable_cuda_graph()
    f.fit(800)
    mesh = extract_mesh_from_sdf_model(f.model_sdf, 128, -0.5, 0.5)
    _, nr = mesh.connected_components()
    assert nr >= 2
    dist = lambda V, s: ((V - torch.tensor(s[0], device="cuda")).norm(dim=1) - s[1]).abs()
    assert int((dist(mesh.V, SMALL) < 0.02).sum()) > 100          # the small sphere was meshed
    nv = mesh.V.shape[0]
    mesh.keep_largest_component()
    assert 1000 < mesh.V.shape[0] < nv and mesh.NV.shape == mesh.V.shape
    assert float(dist(mesh.V, BIG).max()) < 0.02, float(dist(mesh.V, BIG).max())
    assert mesh.connected_components()[1] == 1
    V, F = mesh.V.cpu().numpy(), mesh.F.cpu().numpy()
    assert C.closed_and_oriented(F, len(V)) and C.euler_characteristic(F) == 2
