"""Vectorised numpy oracle of the marching cubes of csrc/marching_cubes.cu (test infrastructure, CPU only).

It builds its own triangle table from the rule alone and follows the same canonical order, so the GPU output is compared with it bit for
bit and in order:
  - a corner is inside when value < threshold (NaN and equality are outside);
  - corner c sits at (c & 1, c >> 1 & 1, c >> 2 & 1); edge 4 a + m runs along axis a, bits 0 and 1 of m are the offsets along the other two
    axes, lower axis first;
  - on each cube face the crossing edges are joined by segments; a face with 4 crossings cuts off its two inside corners;
  - the segments close into loops, taken in the order of their smallest edge; each starts there, runs so that its right-hand normal
    points from inside to outside, and is fanned from its first edge;
  - one vertex per crossing grid edge at the corner plus t = (thr - f_lo) / (f_hi - f_lo) in float32 along the edge axis;
  - vertices slice by slice: in-plane axis-1 edges, in-plane axis-2 edges (row-major in (j, k)), then the axis-0 edges to the next slice;
    faces cell by cell in row-major (i, j, k), table order within a cell.
"""
import numpy as np


def _corner_pos(c):
    return np.array([c & 1, c >> 1 & 1, c >> 2 & 1])


def _edge_corners(e):
    """edge 4 a + m -> (lower corner, upper corner) as corner numbers"""
    a, m = divmod(e, 4)
    others = [x for x in range(3) if x != a]
    p = np.zeros(3, dtype=int)
    p[others[0]], p[others[1]] = m & 1, m >> 1 & 1
    lo = int(p[0] + 2 * p[1] + 4 * p[2])
    return lo, lo + (1 << a)


EDGE_CORNERS = [_edge_corners(e) for e in range(12)]
_EDGE_BY_CORNERS = {frozenset(ec): e for e, ec in enumerate(EDGE_CORNERS)}


def _faces():
    """the six cube faces: (axis, side, corners in cyclic order)"""
    out = []
    for a in range(3):
        u, v = [x for x in range(3) if x != a]
        for s in (0, 1):
            cyc = []
            for pu, pv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[a], p[u], p[v] = s, pu, pv
                cyc.append(p[0] + 2 * p[1] + 4 * p[2])
            out.append((a, s, cyc))
    return out


FACES = _faces()


def _segments(cfg):
    """-> [(edge, edge, face normal (int vector), inside corner the segment cuts off or keeps on its side)]"""
    segs = []
    for a, s, cyc in FACES:
        ins = [cfg >> c & 1 for c in cyc]
        edges = [_EDGE_BY_CORNERS[frozenset((cyc[k], cyc[(k + 1) % 4]))] for k in range(4)]
        crossing = [k for k in range(4) if ins[k] != ins[(k + 1) % 4]]
        normal = np.zeros(3, dtype=int)
        normal[a] = 2 * s - 1
        if len(crossing) == 2:
            ref = next(cyc[k] for k in range(4) if ins[k])
            segs.append((edges[crossing[0]], edges[crossing[1]], normal, ref))
        elif len(crossing) == 4:
            for k in range(4):
                if ins[k]:
                    segs.append((edges[(k + 3) % 4], edges[k], normal, cyc[k]))
    return segs


def _mid2(e):
    lo, hi = EDGE_CORNERS[e]
    return _corner_pos(lo) + _corner_pos(hi)


def _inside_on_right(ea, eb, normal, ref):
    """going ea -> eb on a face, the inside corner `ref` lies to the right seen from outside the cube"""
    d = _mid2(eb) - _mid2(ea)
    r = 2 * _corner_pos(ref) - _mid2(ea)
    return int(np.dot(np.cross(d, r), normal)) < 0


def cell_triangles(cfg):
    """triangles of one corner configuration (bit c = corner c inside): list of (e0, e1, e2)"""
    segs = _segments(cfg)
    adj = {}
    for ea, eb, normal, ref in segs:
        adj.setdefault(ea, []).append((eb, normal, ref))
        adj.setdefault(eb, []).append((ea, normal, ref))
    assert all(len(v) == 2 for v in adj.values())
    tris, done = [], set()
    for start in sorted(adj):
        if start in done:
            continue
        first = next(nb for nb, normal, ref in adj[start] if _inside_on_right(start, nb, normal, ref))
        loop, prev, cur = [start], start, first
        while cur != start:
            loop.append(cur)
            nxt = [nb for nb, _, _ in adj[cur] if nb != prev]
            prev, cur = cur, nxt[0]
        done.update(loop)
        tris += [(loop[0], loop[k], loop[k + 1]) for k in range(1, len(loop) - 1)]
    return tris


TABLE = [cell_triangles(cfg) for cfg in range(256)]


def marching_cubes(volume, threshold=0.0):
    """volume float32 [N0, N1, N2] (each >= 2) -> (verts float32 [V,3] in index space, faces int32 [F,3])"""
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    thr = np.float32(threshold)
    N0, N1, N2 = vol.shape
    ins = vol < thr
    # crossing edges per kind: axis 1 / axis 2 in every slice, axis 0 between slices
    x1 = ins[:, :-1, :] != ins[:, 1:, :]
    x2 = ins[:, :, :-1] != ins[:, :, 1:]
    x0 = ins[:-1] != ins[1:]
    c1 = x1.reshape(N0, -1).sum(1)
    c2 = x2.reshape(N0, -1).sum(1)
    c0 = np.append(x0.reshape(N0 - 1, -1).sum(1), 0)
    per_slice = np.stack([c1, c2, c0], 1).reshape(-1)            # slice-major: axis 1, axis 2, axis 0
    starts = (np.cumsum(per_slice) - per_slice).reshape(N0, 3)

    def ids(x, start):
        flat = x.reshape(x.shape[0], -1)
        r = np.cumsum(flat, 1) - 1 + start[:, None]
        return np.where(flat, r, -1).reshape(x.shape)

    id1, id2, id0 = ids(x1, starts[:, 0]), ids(x2, starts[:, 1]), ids(x0, starts[:N0 - 1, 2])
    nv = int(per_slice.sum())
    verts = np.zeros((nv, 3), dtype=np.float32)

    def place(x, idg, axis, lo, hi):
        i, j, k = np.nonzero(x)
        f_lo, f_hi = lo[i, j, k], hi[i, j, k]
        t = (thr - f_lo) / (f_hi - f_lo)
        c = [i.astype(np.float32), j.astype(np.float32), k.astype(np.float32)]
        c[axis] = c[axis] + t
        verts[idg[i, j, k]] = np.stack(c, 1)

    with np.errstate(invalid="ignore", divide="ignore"):
        place(x1, id1, 1, vol[:, :-1, :], vol[:, 1:, :])
        place(x2, id2, 2, vol[:, :, :-1], vol[:, :, 1:])
        place(x0, id0, 0, vol[:-1], vol[1:])

    cube = np.zeros((N0 - 1, N1 - 1, N2 - 1), dtype=np.int64)
    for c in range(8):
        di, dj, dk = _corner_pos(c)
        cube |= ins[di:N0 - 1 + di, dj:N1 - 1 + dj, dk:N2 - 1 + dk].astype(np.int64) << c
    ntri = np.array([len(t) for t in TABLE])
    cube_flat = cube.reshape(-1)
    cells = np.nonzero(ntri[cube_flat])[0]
    if cells.size == 0:
        return verts, np.zeros((0, 3), dtype=np.int32)
    ci, cj, ck = np.unravel_index(cells, cube.shape)
    # global vertex id of each of the 12 edges of the non-empty cells
    eid = np.empty((cells.size, 12), dtype=np.int64)
    for e in range(12):
        a, m = divmod(e, 4)
        b0, b1 = m & 1, m >> 1 & 1
        if a == 0:
            eid[:, e] = id0[ci, cj + b0, ck + b1]
        elif a == 1:
            eid[:, e] = id1[ci + b0, cj, ck + b1]
        else:
            eid[:, e] = id2[ci + b0, cj + b1, ck]
    tri_tab = np.full((256, 10, 3), -1, dtype=np.int64)
    for cfg, tris in enumerate(TABLE):
        for t, tri in enumerate(tris):
            tri_tab[cfg, t] = tri
    cfgs = cube_flat[cells]
    n = ntri[cfgs]
    rows = np.repeat(np.arange(cells.size), n)
    slot = np.arange(rows.size) - np.repeat(np.cumsum(n) - n, n)
    edges = tri_tab[cfgs[rows], slot]                            # [F,3] cell edge numbers
    faces = np.take_along_axis(eid[rows], edges, 1)
    assert (faces >= 0).all()
    return verts, faces.astype(np.int32)


def single_cell_volume(cfg, inside=-1.0, outside=1.0):
    """2x2x2 volume whose corner c is inside exactly when bit c of cfg is set"""
    v = np.full((2, 2, 2), outside, dtype=np.float32)
    for c in range(8):
        if cfg >> c & 1:
            v[c & 1, c >> 1 & 1, c >> 2 & 1] = inside
    return v


def edge_is_on_face(ea, eb):
    """two cell edges lie on one cube face"""
    return any(set(EDGE_CORNERS[ea]) | set(EDGE_CORNERS[eb]) <= set(cyc) for _, _, cyc in FACES)

