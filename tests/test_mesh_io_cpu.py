"""Reading meshes without a GPU (Mesh.load on CPU tensors): PLY in ascii and both binary byte orders, float and double coordinates,
normals, skipped properties and elements, quads and pentagons; OBJ with every face form and negative indices; binary and ASCII STL,
including a binary file whose header starts with "solid"; the save_to_file -> load round trip bit for bit; the errors for truncated
files, out-of-range indices, unsupported types and unknown list elements; and remove_duplicate_vertices, remove_unreferenced_verts,
normalize_position, normalize_size, scale_mesh and translate on CPU tensors."""
import struct

import numpy as np
import pytest
import torch

from permuto_sdf_b200.mesh import Mesh

# a unit square (two triangles' worth of quad) and a pentagon next to it
QUAD_V = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [2, 0, 0.5], [3, 0, 0.25], [3.5, 1, 0], [2.5, 2, 0], [2, 1, 0.125]],
                  np.float32)
POLYS = [[0, 1, 2, 3], [4, 5, 6, 7, 8], [0, 2, 1]]
FAN = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7], [4, 7, 8], [0, 2, 1]], np.int32)


def ply_bytes(fmt, V, polys, NV=None, vtype="float", ctype="uchar", itype="int", name="vertex_indices", extra=True):
    """a PLY with an extra uchar property before x, an extra element between vertex and face, and a fixed-size property after the face
    list (all skipped on reading)"""
    bo = {"binary_little_endian": "<", "binary_big_endian": ">"}.get(fmt)
    h = ["ply", "format %s 1.0" % fmt, "comment written by a test", "element vertex %d" % len(V)]
    h += ["property uchar quality"] if extra else []
    h += ["property %s %s" % (vtype, a) for a in "xyz"]
    h += ["property %s %s" % (vtype, a) for a in ("nx", "ny", "nz")] if NV is not None else []
    h += ["element material 2", "property float r", "property short g"] if extra else []
    h += ["element face %d" % len(polys), "property list %s %s %s" % (ctype, itype, name)]
    h += ["property ushort flags"] if extra else []
    head = ("\n".join(h + ["end_header"]) + "\n").encode("ascii")
    rows = [list(v) + (list(NV[i]) if NV is not None else []) for i, v in enumerate(V)]
    if bo is None:
        lines = [" ".join(["7"] * extra + [repr(float(x)) for x in r]) for r in rows]
        lines += ["0.5 3", "1.5 -4"] if extra else []
        lines += [" ".join([str(len(p))] + [str(i) for i in p] + ["9"] * extra) for p in polys]
        return head + ("\n".join(lines) + "\n").encode("ascii")
    t = {"float": "f", "double": "d", "uchar": "B", "ushort": "H", "short": "h", "int": "i", "uint": "I", "char": "b"}
    out = bytearray(head)
    for r in rows:
        out += struct.pack(bo + "B" * extra + t[vtype] * len(r), *([3] * extra + list(map(float, r))))
    if extra:
        out += struct.pack(bo + "fh", 0.5, 3) + struct.pack(bo + "fh", 1.5, -4)
    for p in polys:
        out += struct.pack(bo + t[ctype] + t[itype] * len(p) + "H" * extra, len(p), *p, *([9] * extra))
    return bytes(out)


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data if isinstance(data, bytes) else data.encode("ascii"))
    return str(p)


def load(path, **kw):
    return Mesh.load(path, device="cpu", **kw)


def bits(t):
    return t.numpy().view(np.int32)


# ------------------------------------------------------------------------------------------------ PLY
@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
@pytest.mark.parametrize("vtype", ["float", "double"])
def test_ply_formats_types_and_polygons(tmp_path, fmt, vtype):
    NV = np.eye(3, dtype=np.float32)[np.arange(len(QUAD_V)) % 3]
    m = load(write(tmp_path, "m.ply", ply_bytes(fmt, QUAD_V, POLYS, NV, vtype=vtype)))
    assert m.V.dtype == torch.float32 and m.F.dtype == torch.int32 and m.V.device.type == "cpu"
    assert np.array_equal(m.V.numpy(), QUAD_V) and np.array_equal(m.F.numpy(), FAN) and np.array_equal(m.NV.numpy(), NV)


@pytest.mark.parametrize("ctype,itype,name", [("uchar", "int", "vertex_indices"), ("int", "uint", "vertex_index"),
                                               ("ushort", "uint", "vertex_indices"), ("char", "int", "vertex_index")])
@pytest.mark.parametrize("fmt", ["binary_little_endian", "binary_big_endian", "ascii"])
def test_ply_face_list_types(tmp_path, ctype, itype, name, fmt):
    m = load(write(tmp_path, "m.ply", ply_bytes(fmt, QUAD_V, POLYS, ctype=ctype, itype=itype, name=name, extra=False)))
    assert np.array_equal(m.F.numpy(), FAN) and m.NV is None


def test_ply_many_runs_of_polygon_sizes(tmp_path):
    rng = np.random.default_rng(0)
    V = rng.standard_normal((50, 3)).astype(np.float32)
    polys = [list(rng.integers(0, 50, int(c))) for c in np.repeat(rng.integers(3, 7, 60), rng.integers(1, 200, 60))]
    want = np.concatenate([[[p[0], p[j], p[j + 1]] for j in range(1, len(p) - 1)] for p in polys])
    for fmt in ("binary_little_endian", "ascii"):
        m = load(write(tmp_path, "m.ply", ply_bytes(fmt, V, polys)))
        assert np.array_equal(m.F.numpy(), want)


def test_save_to_file_round_trip_is_bit_for_bit(tmp_path):
    rng = np.random.default_rng(1)
    V = torch.from_numpy((rng.standard_normal((1000, 3)) * 10.0 ** rng.integers(-30, 30, (1000, 1))).astype(np.float32))
    V[0] = torch.tensor([-0.0, float(np.float32(1e-45)), float(np.finfo(np.float32).max)])
    NV = torch.nn.functional.normalize(torch.from_numpy(rng.standard_normal((1000, 3)).astype(np.float32)), dim=1)
    Fc = torch.from_numpy(rng.integers(0, 1000, (3000, 3)).astype(np.int32))
    p = str(tmp_path / "m.ply")
    Mesh(V, Fc, NV).save_to_file(p)
    m = load(p)
    assert np.array_equal(bits(m.V), bits(V)) and np.array_equal(m.F.numpy(), Fc.numpy()) and np.array_equal(bits(m.NV), bits(NV))


def test_ply_errors_name_the_path(tmp_path):
    good = ply_bytes("binary_little_endian", QUAD_V, POLYS)
    for name, data, match in [
            ("truncated.ply", good[:-5], "truncated"),
            ("truncated_vertices.ply", good[:good.index(b"end_header") + 40], "truncated"),
            ("range.ply", ply_bytes("binary_little_endian", QUAD_V, [[0, 1, 9]]), r"outside \[0, 9\)"),
            ("negative.ply", ply_bytes("ascii", QUAD_V, [[0, -1, 2]]), r"outside \[0, 9\)"),
            ("list.ply", good.replace(b"element material 2\nproperty float r",
                                      b"element material 2\nproperty list uchar int r"), "list element 'material'"),
            ("type.ply", good.replace(b"property short g", b"property int128 g"), "property type 'int128'"),
            ("floatidx.ply", ply_bytes("binary_little_endian", QUAD_V, POLYS, itype="float"), "integers expected"),
            ("noend.ply", b"ply\nformat ascii 1.0\nelement vertex 1\n", "end_header")]:
        p = write(tmp_path, name, data)
        with pytest.raises(RuntimeError, match="Mesh.load: " + str(tmp_path) + ".*" + match):
            load(p)


# ------------------------------------------------------------------------------------------------ OBJ
def test_obj_face_forms_and_negative_indices(tmp_path):
    text = "\n".join(["# a comment", "mtllib x.mtl", "o thing"] + ["v %r %r %r" % tuple(map(float, v)) for v in QUAD_V[:4]] +
                     ["vn 0 0 1", "vt 0.5 0.5", "f 1 2 3 4", "g group", "usemtl m",
                      "v %r %r %r 1.0" % tuple(map(float, QUAD_V[4]))] + ["v %r %r %r" % tuple(map(float, v)) for v in QUAD_V[5:]] +
                     ["f 5/1 6/1/1 7//1 -2/1 -1", "f -9//1 -7/1/1 -8", "s off", "l 1 2"]) + "\n"
    m = load(write(tmp_path, "m.obj", text))
    assert np.array_equal(m.V.numpy(), QUAD_V) and np.array_equal(m.F.numpy(), FAN) and m.NV is None


def test_obj_errors(tmp_path):
    with pytest.raises(RuntimeError, match="Mesh.load: .*range.obj.*outside"):
        load(write(tmp_path, "range.obj", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 4\n"))
    with pytest.raises(RuntimeError, match="Mesh.load: .*bad.obj.*line 2"):
        load(write(tmp_path, "bad.obj", "v 0 0 0\nv 1 0\n"))


# ------------------------------------------------------------------------------------------------ STL
def stl_binary(tris, header=b"binary stl"):
    rec = np.zeros(len(tris), dtype=[("n", "<f4", (3,)), ("v", "<f4", (3, 3)), ("attr", "<u2")])
    rec["v"] = tris
    return header.ljust(80, b" ") + struct.pack("<I", len(tris)) + rec.tobytes()


def stl_ascii(tris):
    out = ["solid thing"]
    for t in tris:
        out += ["  facet normal 0 0 1", "    outer loop"] + ["      vertex %r %r %r" % tuple(map(float, v)) for v in t]
        out += ["    endloop", "  endfacet"]
    return "\n".join(out + ["endsolid thing"]) + "\n"


TRIS = QUAD_V[FAN]


@pytest.mark.parametrize("kind", ["binary", "binary_solid", "ascii"])
def test_stl_welded_and_soup(tmp_path, kind):
    data = {"binary": lambda: stl_binary(TRIS), "binary_solid": lambda: stl_binary(TRIS, b"solid but binary"),
            "ascii": lambda: stl_ascii(TRIS)}[kind]()
    p = write(tmp_path, "m.stl", data)
    soup = load(p, weld=False)
    assert np.array_equal(soup.V.numpy(), TRIS.reshape(-1, 3)) and np.array_equal(soup.F.numpy(), np.arange(18).reshape(6, 3))
    m = load(p)
    # welded: first occurrences in order, FAN renumbered by first appearance
    order = list(dict.fromkeys(FAN.reshape(-1).tolist()))
    assert np.array_equal(m.V.numpy(), QUAD_V[order]) and m.NV is None
    new = {v: i for i, v in enumerate(order)}
    assert np.array_equal(m.F.numpy(), np.vectorize(new.get)(FAN))


def test_stl_errors(tmp_path):
    data = stl_binary(TRIS)
    with pytest.raises(RuntimeError, match="Mesh.load: .*short.stl.*neither a binary STL"):
        load(write(tmp_path, "short.stl", data[:-7]))
    with pytest.raises(RuntimeError, match="Mesh.load: .*cut.stl.*truncated ASCII STL"):
        load(write(tmp_path, "cut.stl", stl_ascii(TRIS)[:-60]))
    with pytest.raises(RuntimeError, match="Mesh.load: .*nothing.xyz.*cannot tell the format"):
        load(write(tmp_path, "nothing.xyz", "1 2 3\n"))
    with pytest.raises(RuntimeError, match="Mesh.load: .*missing.ply"):
        load(str(tmp_path / "missing.ply"))


# ------------------------------------------------------------------------------------------------ small operations
def test_remove_duplicate_vertices():
    V = torch.tensor([[0, 0, 0], [1, 0, 0], [-0.0, 0, 0], [0, 1, 0], [1, 0, 0], [5, 5, 5], [0, 1, 0]], dtype=torch.float32)
    NV = torch.arange(21, dtype=torch.float32).reshape(7, 3)
    Fc = torch.tensor([[2, 4, 6], [0, 1, 3], [0, 2, 1], [4, 3, 5]], dtype=torch.int32)
    m = Mesh(V, Fc, NV).remove_duplicate_vertices()
    assert torch.equal(m.V, V[[0, 1, 3, 5]]) and torch.equal(m.NV, NV[[0, 1, 3, 5]])
    assert m.F.tolist() == [[0, 1, 2], [0, 1, 2], [1, 2, 3]]          # [0, 2, 1] now repeats vertex 0 and is dropped
    with pytest.raises(RuntimeError, match="not finite"):
        Mesh(torch.tensor([[0, float("nan"), 0]]), torch.zeros(0, 3, dtype=torch.int32)).remove_duplicate_vertices()


def test_remove_unreferenced_verts():
    V = torch.arange(18, dtype=torch.float32).reshape(6, 3)
    m = Mesh(V, torch.tensor([[5, 1, 3], [3, 1, 4]], dtype=torch.int32), V + 100).remove_unreferenced_verts()
    assert torch.equal(m.V, V[[1, 3, 4, 5]]) and torch.equal(m.NV, V[[1, 3, 4, 5]] + 100)
    assert m.F.tolist() == [[3, 0, 1], [1, 0, 2]]


def test_normalize_scale_translate():
    V = torch.tensor([[1, 2, 3], [3, 6, 3], [2, 2, 7]], dtype=torch.float32)
    m = Mesh(V.clone(), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    s = m.normalize_size()
    assert s == 1.0 / 6.0 and torch.equal(m.V, V * np.float32(1.0 / 6.0))
    c = m.normalize_position()
    lo, hi = (V * s).min(0).values, (V * s).max(0).values
    assert torch.equal(c, (lo + hi) / 2)
    assert torch.allclose(m.V.min(0).values, -m.V.max(0).values, rtol=0, atol=1e-7)
    # the calls of train_4d_sdf.py that put a second mesh into the first one's frame, and back
    m2 = Mesh(V.clone(), m.F).scale_mesh(s).translate(-c)
    assert torch.equal(m2.V, m.V)
    m.translate(c).scale_mesh(1.0 / s)
    assert torch.allclose(m.V, V, rtol=1e-6)
