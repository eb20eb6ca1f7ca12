"""Numpy oracle of the quadric decimation and the vertex normals of csrc/mesh_decimate.cu (test infrastructure, CPU only).

It restates the rules of include/psdf_b200.h ("mesh decimation and vertex normals") round by round, with the same fp64 and fp32
operations in the same order, so Mesh.decimate and Mesh.recalculate_normals are compared with it bit for bit. Every round is vectorised
over the candidate half-edges: the faces of a vertex are a padded [V, D] table (D the largest face count), which meshes of some 20 k faces
run through in seconds.
"""
import numpy as np

NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)
MAX_FACES = 64          # an edge with an end in more faces is no candidate


def _valid(F, nv):
    inr = ((F >= 0) & (F < nv)).all(1)
    dis = (F[:, 0] != F[:, 1]) & (F[:, 1] != F[:, 2]) & (F[:, 2] != F[:, 0])
    return inr, inr & dis


def vertex_faces(F, nv):
    """faces of each vertex in ascending order (faces outside [0, nv) or with a repeated vertex left out) -> (A [nv, D] with -1 padding,
    face counts [nv])"""
    _, ok = _valid(F, nv)
    f = np.nonzero(ok)[0]
    v = F[f].reshape(-1)
    fv = np.repeat(f, 3)
    order = np.lexsort((fv, v))
    v, fv = v[order], fv[order]
    deg = np.bincount(v, minlength=nv)
    start = np.concatenate([[0], np.cumsum(deg)[:-1]])
    slot = np.arange(v.size) - start[v]
    A = np.full((nv, max(1, int(deg.max()) if nv else 1)), -1, dtype=np.int64)
    A[v, slot] = fv
    return A, deg


def _around(F, A, s):
    """faces of the vertices s: (face ids [n, D] clipped to 0, valid [n, D], vertices [n, D, 3], next and previous corner of s)"""
    fa = A[s]
    ok = fa >= 0
    fa = np.where(ok, fa, 0)
    T = F[fa]
    pos = np.argmax(T == s[:, None, None], axis=2)
    nx = np.take_along_axis(T, ((pos + 1) % 3)[..., None], 2)[..., 0]
    pv = np.take_along_axis(T, ((pos + 2) % 3)[..., None], 2)[..., 0]
    return fa, ok, T, nx, pv


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def face_quadrics(V, F):
    """[F, 10] area-weighted plane quadrics, and whether the face has non-zero area"""
    p = V[F].astype(np.float64)
    N = _cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    l = np.sqrt(_dot(N, N))
    nz = l > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        n = N / l[:, None]
        d = -((n[:, 0] * p[:, 0, 0] + n[:, 1] * p[:, 0, 1]) + n[:, 2] * p[:, 0, 2])
        w = l * 0.5
        x, y, z = n[:, 0], n[:, 1], n[:, 2]
        q = np.stack([w * (x * x), w * (x * y), w * (x * z), w * (x * d), w * (y * y), w * (y * z), w * (y * d), w * (z * z), w * (z * d),
                      w * (d * d)], 1)
    return q, nz


def quadric_error(Q, p):
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r0 = ((Q[:, 0] * x + Q[:, 1] * y) + Q[:, 2] * z) + Q[:, 3]
    r1 = ((Q[:, 1] * x + Q[:, 4] * y) + Q[:, 5] * z) + Q[:, 6]
    r2 = ((Q[:, 2] * x + Q[:, 5] * y) + Q[:, 7] * z) + Q[:, 8]
    r3 = ((Q[:, 3] * x + Q[:, 6] * y) + Q[:, 8] * z) + Q[:, 9]
    return ((x * r0 + y * r1) + z * r2) + r3


def place(Q, pa, pb):
    """positions (float32) and errors of unlocked pairs"""
    c00 = Q[:, 4] * Q[:, 7] - Q[:, 5] * Q[:, 5]
    c01 = Q[:, 2] * Q[:, 5] - Q[:, 1] * Q[:, 7]
    c02 = Q[:, 1] * Q[:, 5] - Q[:, 4] * Q[:, 2]
    c11 = Q[:, 0] * Q[:, 7] - Q[:, 2] * Q[:, 2]
    c12 = Q[:, 1] * Q[:, 2] - Q[:, 0] * Q[:, 5]
    c22 = Q[:, 0] * Q[:, 4] - Q[:, 1] * Q[:, 1]
    det = (Q[:, 0] * c00 + Q[:, 1] * c01) + Q[:, 2] * c02
    tr = (Q[:, 0] + Q[:, 4]) + Q[:, 7]
    good = np.abs(det) > 1e-12 * ((tr * tr) * tr)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        x = np.stack([-(((c00 * Q[:, 3] + c01 * Q[:, 6]) + c02 * Q[:, 8]) / det),
                      -(((c01 * Q[:, 3] + c11 * Q[:, 6]) + c12 * Q[:, 8]) / det),
                      -(((c02 * Q[:, 3] + c12 * Q[:, 6]) + c22 * Q[:, 8]) / det)], 1)
        a, b = pa.astype(np.float64), pb.astype(np.float64)
        m = (a + b) * 0.5
        dx, e = x - m, b - a
        good &= _dot(dx, dx) <= _dot(e, e)
        xs = x.astype(np.float32)
    pm = (pa + pb) * np.float32(0.5)
    p, cost = pa.copy(), quadric_error(Q, pa.astype(np.float64))
    for alt in (pb, pm):
        c = quadric_error(Q, alt.astype(np.float64))
        better = c < cost
        p[better], cost[better] = alt[better], c[better]
    p[good] = xs[good]
    cost[good] = quadric_error(Q[good], xs[good].astype(np.float64))
    return p, cost


def _faces_hold(V, F, A, s, p, f, g):
    """no face of s other than f and g flips or becomes degenerate when s moves to p"""
    fa, ok, T, _, _ = _around(F, A, s)
    ok &= (fa != f[:, None]) & (fa != g[:, None])
    P = V[T].astype(np.float64)
    n0 = _cross(P[:, :, 1] - P[:, :, 0], P[:, :, 2] - P[:, :, 0])
    moved = T == s[:, None, None]
    P = np.where(moved[..., None], p.astype(np.float64)[:, None, None, :], P)
    n1 = _cross(P[:, :, 1] - P[:, :, 0], P[:, :, 2] - P[:, :, 0])
    return (~ok | (_dot(n0, n1) > 0)).all(1)


def candidate_keys(V, F, Q, lock):
    """keys [3F] of every half-edge (NO_KEY for non-candidates and failed checks), and per candidate (a, b, f, g, position, Q sum)"""
    nv = V.shape[0]
    A, deg = vertex_faces(F, nv)
    c = np.arange(3 * F.shape[0])
    f, k = c // 3, c % 3
    u, v, w = F[f, k], F[f, (k + 1) % 3], F[f, (k + 2) % 3]
    keys = np.full(c.size, NO_KEY, dtype=np.uint64)
    s = np.nonzero((u < v) & (deg[u] <= MAX_FACES) & (deg[v] <= MAX_FACES))[0]
    fa, ok, _, nxu, pv = _around(F, A, u[s])
    nsame = ((nxu == v[s][:, None]) & ok).sum(1)
    istw = (pv == v[s][:, None]) & ok
    ntwin = istw.sum(1)
    g = fa[np.arange(s.size), np.argmax(istw, 1)]
    keep = (nsame == 1) & (ntwin == 1) & ~(lock[u[s]] & lock[v[s]])
    s, g = s[keep], g[keep]
    us, vs, ws = u[s], v[s], w[s]
    a = np.where(lock[vs], vs, us)
    b = np.where(lock[vs], us, vs)
    Tg = F[g]
    d = np.where((Tg[:, 0] != us) & (Tg[:, 0] != vs), Tg[:, 0], np.where((Tg[:, 1] != us) & (Tg[:, 1] != vs), Tg[:, 1], Tg[:, 2]))
    keep = (ws != d) & (deg[ws] > 3) & (deg[d] > 3)
    # link condition: the corners that follow b in its faces, other than a, that lie in a face of a
    _, okb, _, nxb, _ = _around(F, A, b)
    _, oka, Ta, _, _ = _around(F, A, a)
    Ta = np.where(oka[..., None], Ta, -1).reshape(a.size, -1)
    inA = (nxb[:, :, None] == Ta[:, None, :]).any(2) & okb & (nxb != a[:, None])
    keep &= inA.sum(1) == 2
    s, g, a, b = s[keep], g[keep], a[keep], b[keep]
    Qs = Q[a] + Q[b]
    pa, pb = V[a], V[b]
    la = lock[a]
    p, cost = pa.copy(), quadric_error(Qs, pa.astype(np.float64))
    if (~la).any():
        p[~la], cost[~la] = place(Qs[~la], pa[~la], pb[~la])
    fs = s // 3
    keep = _faces_hold(V, F, A, a, p, fs, g) & _faces_hold(V, F, A, b, p, fs, g)
    s, g, a, b, p, cost, Qs, fs = s[keep], g[keep], a[keep], b[keep], p[keep], cost[keep], Qs[keep], fs[keep]
    cf = np.where(cost > 0, cost, 0.0).astype(np.float32)
    keys[s] = (cf.view(np.uint32).astype(np.uint64) << np.uint64(33)) | s.astype(np.uint64)
    return keys, dict(c=s, a=a, b=b, f=fs, g=g, p=p, Q=Qs), A


def begin(V, F):
    """-> (faces outside [0, V), faces repeating a vertex, Q [V, 10], locks [V])"""
    nv = V.shape[0]
    inr, ok = _valid(F, nv)
    bad, rep = int((~inr).sum()), int((inr & ~ok).sum())
    A, deg = vertex_faces(F, nv)
    lock = np.zeros(nv, dtype=bool)
    Fv = F[ok]
    if Fv.size:
        c = np.arange(3 * Fv.shape[0])
        f, k = c // 3, c % 3
        u, v = Fv[f, k], Fv[f, (k + 1) % 3]
        Fc = np.where(ok[:, None], F, 0)
        _, okk, _, nx, pv = _around(Fc, A, u)
        bad_edge = (((nx == v[:, None]) & okk).sum(1) != 1) | (((pv == v[:, None]) & okk).sum(1) != 1)
        lock[u[bad_edge]] = True
        lock[v[bad_edge]] = True
    Q = np.zeros((nv, 10))
    if Fv.size:
        q, nz = face_quadrics(V, np.where(ok[:, None], F, 0))
        for j in range(A.shape[1]):
            fa = A[:, j]
            m = fa >= 0
            m[m] &= nz[fa[m]]
            Q[m] = Q[m] + q[fa[m]]
    return bad, rep, Q, lock


def one_round(V, F, Q, lock, removed, allowed):
    """one round in place on V, Q, removed -> (new F, chosen, applied)"""
    nv = V.shape[0]
    keys, cand, A = candidate_keys(V, F, Q, lock)
    best = np.full(nv, NO_KEY, dtype=np.uint64)
    kc = keys[cand["c"]]
    np.minimum.at(best, cand["a"], kc)
    np.minimum.at(best, cand["b"], kc)
    best2 = best.copy()
    for j in range(A.shape[1]):
        fa = A[:, j]
        m = fa >= 0
        best2[m] = np.minimum(best2[m], best[F[fa[m]]].min(1))
    c = np.arange(keys.size)
    u, v = F[c // 3, c % 3], F[c // 3, (c % 3 + 1) % 3]
    chosen = np.nonzero((keys != NO_KEY) & (keys == best2[u]) & (keys == best2[v]))[0]
    n = chosen.size
    if n > allowed:
        thr = np.sort(keys[chosen])[allowed - 1]
        chosen = chosen[keys[chosen] <= thr]
    idx = np.searchsorted(cand["c"], chosen)
    a, b, f, g = cand["a"][idx], cand["b"][idx], cand["f"][idx], cand["g"][idx]
    V[a] = cand["p"][idx]
    Q[a] = cand["Q"][idx]
    removed[b] = True
    remap = np.arange(nv)
    remap[b] = a
    drop = np.zeros(F.shape[0], dtype=bool)
    drop[f] = drop[g] = True
    return remap[F[~drop]], n, chosen.size


def decimate(V, F, nr_target_faces):
    """the rounds of Mesh.decimate before the final compaction -> (V [nv,3] float32, F [m,3] int64, removed [nv] bool, rounds)"""
    V = np.array(V, dtype=np.float32).reshape(-1, 3)
    F = np.array(F, dtype=np.int64).reshape(-1, 3)
    removed = np.zeros(V.shape[0], dtype=bool)
    if nr_target_faces >= F.shape[0]:
        return V, F, removed, 0
    bad, rep, Q, lock = begin(V, F)
    if bad or rep:
        raise ValueError("%d faces outside [0, V), %d faces repeating a vertex" % (bad, rep))
    rounds = 0
    while True:
        allowed = (F.shape[0] - nr_target_faces + 1) // 2
        if allowed <= 0:
            break
        F, _, applied = one_round(V, F, Q, lock, removed, allowed)
        rounds += 1
        if applied == 0:
            break
    return V, F, removed, rounds


def normals(V, F):
    """vertex normals [nv,3] float32 of Mesh.recalculate_normals"""
    V = np.asarray(V, dtype=np.float32).reshape(-1, 3)
    F = np.asarray(F, dtype=np.int64).reshape(-1, 3)
    nv = V.shape[0]
    A, _ = vertex_faces(F, nv)
    _, ok = _valid(F, nv)
    p = V[np.where(ok[:, None], F, 0)]
    a, b = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    cr = _cross(a, b)
    n = np.zeros((nv, 3), dtype=np.float32)
    for j in range(A.shape[1]):
        fa = A[:, j]
        m = fa >= 0
        n[m] = n[m] + cr[fa[m]]
    l = np.sqrt(_dot(n, n))
    with np.errstate(invalid="ignore", divide="ignore"):
        out = n / l[:, None]
    out[~(l > 0)] = 0
    return out.astype(np.float32)


def decimate_mesh(V, F, nr_target_faces, with_normals):
    """Mesh(V, F, NV).decimate(nr_target_faces) -> (V, F int32, NV or None, rounds)"""
    Vd, Fd, removed, rounds = decimate(V, F, nr_target_faces)
    if rounds == 0 and nr_target_faces >= np.asarray(F).reshape(-1, 3).shape[0]:
        return Vd, Fd.astype(np.int32), None, 0
    kept = ~removed
    new_id = np.cumsum(kept) - 1
    Vd, Fd = Vd[kept], new_id[Fd].astype(np.int32)
    return Vd, Fd, normals(Vd, Fd) if with_normals else None, rounds
