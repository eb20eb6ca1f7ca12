"""Mesh properties shared by the marching-cubes tests (numpy, host arrays)."""
import numpy as np


def directed_edges(F):
    F = np.asarray(F, dtype=np.int64)
    return np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]])


def _keys(e, n):
    return e[:, 0] * n + e[:, 1]


def closed_and_oriented(F, nv):
    """every directed edge appears once and its reverse appears once"""
    e = directed_edges(F)
    k, r = _keys(e, nv), _keys(e[:, ::-1], nv)
    uk = np.unique(k)
    return uk.size == k.size and np.array_equal(uk, np.unique(r))


def balanced(F, nv):
    """index-closed and consistently oriented, where an edge may be shared by more than two triangles: every directed edge appears as
    often as its reverse"""
    e = directed_edges(F)
    uk, ck = np.unique(_keys(e, nv), return_counts=True)
    ur, cr = np.unique(_keys(e[:, ::-1], nv), return_counts=True)
    return np.array_equal(uk, ur) and np.array_equal(ck, cr)


def euler_characteristic(F):
    F = np.asarray(F, dtype=np.int64)
    e = np.sort(directed_edges(F), 1)
    return np.unique(F).size - np.unique(e, axis=0).shape[0] + F.shape[0]


def signed_volume(V, F):
    v = np.asarray(V, dtype=np.float64)[np.asarray(F, dtype=np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def read_ply(path):
    """the binary little-endian PLY written by Mesh.save_to_file -> (V [n,3], NV [n,3], F [m,3])"""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").split("\n")
    assert header[0] == "ply" and header[1] == "format binary_little_endian 1.0"
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[2])
    nf = int(next(h for h in header if h.startswith("element face")).split()[2])
    props = [h.split()[2] for h in header if h.startswith("property float")]
    assert props == ["x", "y", "z", "nx", "ny", "nz"]
    assert "property list uchar int vertex_indices" in header
    vert = np.frombuffer(data, dtype="<f4", count=6 * nv, offset=end).reshape(nv, 6)
    face = np.frombuffer(data, dtype=[("n", "u1"), ("idx", "<i4", (3,))], count=nf, offset=end + 24 * nv)
    assert (face["n"] == 3).all() and end + 24 * nv + 13 * nf == len(data)
    return vert[:, :3], vert[:, 3:], face["idx"]


def grid(shape):
    return np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")


def sphere_volume(shape, center, radius):
    x, y, z = grid(shape)
    return (np.sqrt((x - center[0]) ** 2 + (y - center[1]) ** 2 + (z - center[2]) ** 2) - radius).astype(np.float32)


def torus_volume(shape, center, R, r):
    x, y, z = grid(shape)
    q = np.sqrt((x - center[0]) ** 2 + (y - center[1]) ** 2) - R
    return (np.sqrt(q ** 2 + (z - center[2]) ** 2) - r).astype(np.float32)


def two_spheres_volume(shape, c0, c1, radius):
    return np.minimum(sphere_volume(shape, c0, radius), sphere_volume(shape, c1, radius))


def random_field(shape, seed, sigma=3.0):
    """smooth noise, positive (outside) on the volume's boundary so the mesh is closed"""
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(seed)
    f = gaussian_filter(rng.standard_normal(shape), sigma)
    f = f / f.std()
    f[[0, -1], :, :] = f[:, [0, -1], :] = f[:, :, [0, -1]] = 1.0
    return f.astype(np.float32)


def pad_outside(v, value=1.0):
    return np.pad(v, 1, constant_values=value).astype(np.float32)
