"""Closest points, pseudonormals, signed distances and surface samples of a triangle mesh by brute force (numpy): the fp32 closest-point
formula of include/psdf_b200.h (Ericson's region test with triple-product areas and guarded divisions, each operation rounded as written) over every face, so that
csrc/mesh_distance.cu's dist2, face and bary can be compared bit for bit; the angle-weighted pseudonormals in fp64; the SplitMix64 surface
samples of psdf_mesh_sample_surface; and an fp64 mesh distance from given samples."""
import numpy as np

f32 = np.float32
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dist2(p, q):
    d = p - q
    return dot(d, d)


def _along(x, e, t):
    return x + t[..., None] * e


def nearest_edge(p, a, b, c):
    """the nearest of the edges ab, bc, ca (the first with the smallest dist2) -> (dist2, bary [..., 3])"""
    best, bary = None, None
    for x, y, k in ((a, b, 0), (b, c, 1), (c, a, 2)):
        e = y - x
        ee = dot(e, e)
        t = np.where(ee > 0, dot(p - x, e) / np.where(ee > 0, ee, f32(1)), f32(0))
        t = np.minimum(np.maximum(t, f32(0)), f32(1))
        d2 = _dist2(p, _along(x, e, t))
        w = np.zeros(d2.shape + (3,), f32)
        w[..., k] = f32(1) - t
        w[..., (k + 1) % 3] = t
        if best is None:
            best, bary = d2, w
        else:
            take = d2 < best
            best, bary = np.where(take, d2, best), np.where(take[..., None], w, bary)
    return best, bary


def closest_on_triangle(p, a, b, c):
    """the formula of include/psdf_b200.h for every broadcast pair of points p [..., 3] and faces (a, b, c [..., 3]) -> (dist2 [...],
    bary [..., 3]), fp32"""
    p, a, b, c = (np.asarray(x, f32) for x in (p, a, b, c))
    shape = np.broadcast_shapes(p.shape, a.shape, b.shape, c.shape)
    p, a, b, c = (np.broadcast_to(x, shape) for x in (p, a, b, c))
    with np.errstate(all="ignore"):
        ab, ac = b - a, c - a
        n = cross(ab, ac)
        degenerate = (n[..., 0] == 0) & (n[..., 1] == 0) & (n[..., 2] == 0)
        ap = p - a
        d1, d2 = dot(ab, ap), dot(ac, ap)
        bp = p - b
        d3, d4 = dot(ab, bp), dot(ac, bp)
        vc = dot(n, cross(ap, bp))
        eab = d1 - d3
        cp = p - c
        d5, d6 = dot(ab, cp), dot(ac, cp)
        vb = dot(n, cross(cp, ap))
        eac = d2 - d6
        va = dot(n, cross(bp, cp))
        e43, e56 = d4 - d3, d5 - d6
        ebc = e43 + e56
        den = (va + vb) + vc
        vi, wi = vb / den, vc / den
        v_ab = d1 / eab
        w_ac = d2 / eac
        w_bc = e43 / ebc
        one, zero = f32(1), f32(0)
        z = np.zeros(shape[:-1], f32)
        cases = [  # (condition, dist2, bary), the first that holds
            (degenerate, None, None),
            ((d1 <= 0) & (d2 <= 0), _dist2(p, a), (z + one, z, z)),
            ((d3 >= 0) & (d4 <= d3), _dist2(p, b), (z, z + one, z)),
            ((vc <= 0) & (d1 >= 0) & (d3 <= 0) & (eab > 0), _dist2(p, _along(a, ab, v_ab)), (one - v_ab, v_ab, z)),
            ((d6 >= 0) & (d5 <= d6), _dist2(p, c), (z, z, z + one)),
            ((vb <= 0) & (d2 >= 0) & (d6 <= 0) & (eac > 0), _dist2(p, _along(a, ac, w_ac)), (one - w_ac, z, w_ac)),
            ((va <= 0) & (e43 >= 0) & (e56 >= 0) & (ebc > 0), _dist2(p, _along(b, c - b, w_bc)), (z, one - w_bc, w_bc)),
        ]
        e_d2, e_bary = nearest_edge(p, a, b, c)
        # interior: the nearest edge instead when it is strictly closer
        i_d2 = _dist2(p, _along(_along(a, ab, vi), ac, wi))
        closer = e_d2 < i_d2
        cases.append(((den > 0) & (vi >= 0) & (wi >= 0) & (vi + wi <= 1), np.where(closer, e_d2, i_d2),
                      tuple(np.where(closer, e_bary[..., k], x) for k, x in enumerate(((one - vi) - wi, vi, wi)))))
        out_d2, out_bary = e_d2.copy(), e_bary.copy()
        done = np.zeros(shape[:-1], bool)
        for cond, d2_, w in cases:
            take = cond & ~done
            if d2_ is not None:
                out_d2 = np.where(take, d2_, out_d2)
                out_bary = np.where(take[..., None], np.stack(w, -1).astype(f32), out_bary)
            done |= cond
    return out_d2.astype(f32), out_bary.astype(f32)


def valid_faces(F):
    F = np.asarray(F, np.int64).reshape(-1, 3)
    return (F[:, 0] != F[:, 1]) & (F[:, 1] != F[:, 2]) & (F[:, 2] != F[:, 0])


def closest_points(V, F, points, chunk=1 << 22):
    """brute force over every face -> (dist2 [P] float32, face [P] int32, bary [P,3] float32): the smallest dist2 over the faces with
    three distinct indices, ties to the smallest face index; none: (+inf, -1, 0)"""
    V, F = np.asarray(V, f32), np.asarray(F, np.int64).reshape(-1, 3)
    pts = np.asarray(points, f32).reshape(-1, 3)
    P = pts.shape[0]
    d2 = np.full(P, np.inf, f32)
    face = np.full(P, -1, np.int32)
    bary = np.zeros((P, 3), f32)
    keep = np.flatnonzero(valid_faces(F))
    if keep.size == 0:
        return d2, face, bary
    a, b, c = V[F[keep, 0]], V[F[keep, 1]], V[F[keep, 2]]
    step = max(1, chunk // keep.size)
    for s in range(0, P, step):
        p = pts[s:s + step, None, :]
        D, B = closest_on_triangle(p, a[None], b[None], c[None])
        j = np.argmin(D, 1)                                     # the first of equal minima: the smallest face index
        r = np.arange(D.shape[0])
        m = D[r, j]
        ok = m < np.inf
        d2[s:s + step] = np.where(ok, m, np.inf)
        face[s:s + step] = np.where(ok, keep[j], -1)
        bary[s:s + step] = np.where(ok[:, None], B[r, j], 0)
    return d2, face, bary


def pseudonormals(V, F):
    """fp64 angle-weighted pseudonormals -> (face_n [F,3] unit, vert_n [V,3], edge_n [F,3,3]) as the header defines them, faces that
    repeat a vertex left out"""
    V, F = np.asarray(V, np.float64), np.asarray(F, np.int64).reshape(-1, 3)
    ok = valid_faces(F)
    p = V[F]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    fn = np.where((ln > 0) & ok[:, None], n / np.where(ln > 0, ln, 1), 0)
    vn = np.zeros_like(V)
    for k in range(3):
        e1 = p[:, (k + 1) % 3] - p[:, k]
        e2 = p[:, (k + 2) % 3] - p[:, k]
        ang = np.arctan2(np.linalg.norm(np.cross(e1, e2), axis=1), np.einsum("ij,ij->i", e1, e2))
        np.add.at(vn, F[ok, k], (ang[:, None] * fn)[ok])
    key = lambda u, v: np.minimum(u, v) * max(V.shape[0], 1) + np.maximum(u, v)
    ek = np.stack([key(F[:, k], F[:, (k + 1) % 3]) for k in range(3)], 1)        # [F,3]
    uk, inv = np.unique(ek[ok].reshape(-1), return_inverse=True)
    sums = np.zeros((uk.size, 3))
    np.add.at(sums, inv, np.repeat(fn[ok], 3, 0))
    en = np.zeros((F.shape[0], 3, 3))
    en[ok] = sums[inv].reshape(-1, 3, 3)
    return fn, vn, en


def feature_normal(face_n, vert_n, edge_n, F, face, bary):
    """the pseudonormal of the feature the weights name (two zeros: a vertex, one: an edge, none: the face) for each query [P,3]"""
    F = np.asarray(F, np.int64).reshape(-1, 3)
    f = np.asarray(face, np.int64)
    z = np.asarray(bary) == 0
    nz = z.sum(1)
    out = face_n[f].copy()
    vi = np.argmax(~z, 1)
    m = nz == 2
    out[m] = vert_n[F[f[m], vi[m]]]
    ek = np.where(z[:, 2], 0, np.where(z[:, 0], 1, 2))
    m = nz == 1
    out[m] = edge_n[f[m], ek[m]]
    return out


def signed_cos(V, F, points, face, bary):
    """fp64 cosine of the angle between p - q and n, the pseudonormal of the closest feature (q from the weights, n from the fp64
    pseudonormals); 0 where either is zero -> [P]. Its sign is the sign of signed_distance; its size says how clear that sign is."""
    V, F = np.asarray(V, np.float64), np.asarray(F, np.int64).reshape(-1, 3)
    fn, vn, en = pseudonormals(V, F)
    f = np.asarray(face, np.int64)
    q = np.einsum("pk,pkj->pj", np.asarray(bary, np.float64), V[F[f]])
    d = np.asarray(points, np.float64) - q
    n = feature_normal(fn, vn, en, F, f, bary)
    ln = np.linalg.norm(d, axis=1) * np.linalg.norm(n, axis=1)
    return np.where(ln > 0, np.einsum("pj,pj->p", d, n) / np.where(ln > 0, ln, 1), 0)


def splitmix64(seed, n):
    """output n (uint64 array) of SplitMix64 seeded with seed"""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (np.asarray(n, np.uint64) + np.uint64(1)) * _GOLDEN
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def sample_surface(V, F, cdf, N, seed):
    """the samples of psdf_mesh_sample_surface -> (points [N,3] float32, face [N] int32)"""
    V, F = np.asarray(V, f32), np.asarray(F, np.int64).reshape(-1, 3)
    cdf = np.asarray(cdf, np.float64)
    n = np.arange(N, dtype=np.uint64) * np.uint64(3)
    total = cdf[-1]
    u0 = (splitmix64(seed, n) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 * total
    face = np.searchsorted(cdf, u0, side="right")
    top = ~(u0 < total)
    face[top] = np.searchsorted(cdf, total, side="left")
    r1 = (splitmix64(seed, n + np.uint64(1)) >> np.uint64(40)).astype(f32) * f32(2.0 ** -24)
    r2 = (splitmix64(seed, n + np.uint64(2)) >> np.uint64(40)).astype(f32) * f32(2.0 ** -24)
    s = np.sqrt(r1)
    w = [f32(1) - s, s * (f32(1) - r2), s * r2]
    p = V[F[face]]
    pts = (w[0][:, None] * p[:, 0] + w[1][:, None] * p[:, 1]) + w[2][:, None] * p[:, 2]
    return pts.astype(f32), face.astype(np.int32)


def point_mesh_distance64(V, F, points):
    """fp64 unsigned distance from each point to the faces (brute force, exact projection onto each triangle) -> [P]"""
    V, F = np.asarray(V, np.float64), np.asarray(F, np.int64).reshape(-1, 3)
    F = F[valid_faces(F)]
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    a, b, c = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    out = np.empty(pts.shape[0])
    step = max(1, (1 << 21) // max(F.shape[0], 1))
    for s in range(0, pts.shape[0], step):
        d2, _ = closest_on_triangle64(pts[s:s + step, None], a[None], b[None], c[None])
        out[s:s + step] = np.sqrt(d2.min(1))
    return out


def closest_on_triangle64(p, a, b, c):
    """the same region test in fp64 (the reference for mesh_distance's accuracy, not for bits)"""
    p, a, b, c = np.broadcast_arrays(*(np.asarray(x, np.float64) for x in (p, a, b, c)))
    return _closest64(p, a, b, c)


def _closest64(p, a, b, c):
    with np.errstate(all="ignore"):
        d2 = None
        # the nearest edge always bounds the answer; the interior projection replaces it when it lands inside
        for x, y in ((a, b), (b, c), (c, a)):
            e = y - x
            ee = dot(e, e)
            t = np.clip(np.where(ee > 0, dot(p - x, e) / np.where(ee > 0, ee, 1), 0), 0, 1)
            d = _dist2(p, x + t[..., None] * e)
            d2 = d if d2 is None else np.minimum(d2, d)
        n = cross(b - a, c - a)
        nn = dot(n, n)
        h = np.where(nn > 0, dot(p - a, n) / np.where(nn > 0, nn, 1), 0)
        q = p - h[..., None] * n
        u = dot(cross(b - q, c - q), n)
        v = dot(cross(c - q, a - q), n)
        w = dot(cross(a - q, b - q), n)
        inside = (nn > 0) & (u >= 0) & (v >= 0) & (w >= 0)
        d2 = np.where(inside, np.minimum(d2, _dist2(p, q)), d2)
    return d2, None


def mesh_distance64(Va, Fa, Vb, Fb, samples_a, samples_b):
    """fp64 accuracy (samples of a to b), completeness (samples of b to a), chamfer and hausdorff from given samples"""
    da = point_mesh_distance64(Vb, Fb, samples_a)
    db = point_mesh_distance64(Va, Fa, samples_b)
    acc, comp = float(da.mean()), float(db.mean())
    return {"accuracy": acc, "completeness": comp, "chamfer": (acc + comp) / 2, "hausdorff": float(max(da.max(), db.max()))}
