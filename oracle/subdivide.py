"""Numpy oracle of the midpoint and Loop subdivision of csrc/mesh_subdivide.cu (test infrastructure, CPU only).

It restates the rules of include/psdf_b200.h ("mesh subdivision") round by round, with the same fp32 operations in the same order, so
Mesh.upsample is compared with it bit for bit. Each round is vectorised: the edges are the corners sorted by (edge, corner id), and the
Loop rule for the old vertices runs over a padded [V, D] table of each vertex's distinct neighbours (D the largest count), which meshes of
some 20 k faces run through in well under a second.
"""
import numpy as np

from .decimate import _valid

F32 = np.float32


def edges(F, nv):
    """-> (own [3F]: the smallest corner id of each corner's edge, -1 at the corners of bad faces; count [3F]: the faces of that edge;
    other [3F]: at an owning corner of an interior edge, the third vertex of the edge's other face, else -1; pos [3F]: exclusive prefix of
    the owning corners; E)"""
    nc = 3 * F.shape[0]
    _, ok = _valid(F, nv)
    c = np.arange(nc)
    f, k = c // 3, c % 3
    u, v = F[f, k], F[f, (k + 1) % 3]
    own = np.full(nc, -1, dtype=np.int64)
    count = np.zeros(nc, dtype=np.int64)
    other = np.full(nc, -1, dtype=np.int64)
    cv = c[ok[f]]
    key = np.minimum(u[cv], v[cv]) * np.int64(max(nv, 1)) + np.maximum(u[cv], v[cv])
    order = np.lexsort((cv, key))
    cs, ks = cv[order], key[order]
    start = np.ones(cs.size, dtype=bool)
    start[1:] = ks[1:] != ks[:-1]
    gid = np.cumsum(start) - 1
    first = np.nonzero(start)[0]
    sizes = np.diff(np.append(first, cs.size))
    own[cs] = cs[first[gid]]
    count[cs] = sizes[gid]
    two = first[sizes == 2]
    c2 = cs[two + 1]
    other[cs[two]] = F[c2 // 3, (c2 % 3 + 2) % 3]
    owner = own == c
    pos = np.cumsum(owner) - owner
    return own, count, other, pos, int(owner.sum())


def _loop_even(V, F, ok):
    """the Loop rule for the old vertices -> positions [nv, 3] float32"""
    nv = V.shape[0]
    Fv = F[ok]
    u = np.concatenate([Fv[:, 0], Fv[:, 1], Fv[:, 2], Fv[:, 1], Fv[:, 2], Fv[:, 0]])
    w = np.concatenate([Fv[:, 1], Fv[:, 2], Fv[:, 0], Fv[:, 0], Fv[:, 1], Fv[:, 2]])
    pairs, mult = np.unique(np.stack([u, w], 1), axis=0, return_counts=True) if u.size else (np.zeros((0, 2), np.int64), np.zeros(0, np.int64))
    pu, pw = pairs[:, 0], pairs[:, 1]
    n = np.bincount(pu, minlength=nv)
    crease = mult != 2
    k = np.bincount(pu, weights=crease, minlength=nv).astype(np.int64)
    start = np.concatenate([[0], np.cumsum(n)[:-1]])
    slot = np.arange(pu.size) - start[pu]
    D = max(1, int(n.max()) if nv else 1)
    N = np.full((nv, D), -1, dtype=np.int64)
    N[pu, slot] = pw
    s = np.zeros((nv, 3), dtype=F32)
    for j in range(D):
        m = N[:, j] >= 0
        s[m] = s[m] + V[N[m, j]]
    out = V.copy()
    i0 = np.nonzero((n > 0) & (k == 0))[0]
    nn = n[i0]
    beta = np.where(nn == 3, F32(0.1875), F32(3.0) / (8 * nn).astype(F32)).astype(F32)
    wv = (F32(1.0) - nn.astype(F32) * beta).astype(F32)
    out[i0] = wv[:, None] * V[i0] + beta[:, None] * s[i0]
    # k = 2: the two crease neighbours in ascending order
    cp = np.nonzero(crease)[0]
    cu = pu[cp]
    firsts = np.ones(cp.size, dtype=bool)
    firsts[1:] = cu[1:] != cu[:-1]
    i2 = np.nonzero(k == 2)[0]
    fi = np.nonzero(firsts)[0]
    a_of = np.full(nv, -1, dtype=np.int64)
    b_of = np.full(nv, -1, dtype=np.int64)
    a_of[cu[fi]] = pw[cp[fi]]
    nxt = fi + 1
    has = nxt < cp.size
    b_of[cu[fi[has]]] = pw[cp[nxt[has]]]
    out[i2] = F32(0.75) * V[i2] + F32(0.125) * (V[a_of[i2]] + V[b_of[i2]])
    return out


def one_round(V, F, smooth):
    """one round -> (V [nv + E, 3] float32, F [4 nf, 3] int64); raises on bad faces"""
    nv, nf = V.shape[0], F.shape[0]
    inr, ok = _valid(F, nv)
    if not ok.all():
        raise ValueError("%d faces outside [0, V), %d faces repeating a vertex" % (int((~inr).sum()), int((inr & ~ok).sum())))
    own, count, other, pos, E = edges(F, nv)
    c = np.arange(3 * nf)
    f, k = c // 3, c % 3
    oc = np.nonzero(own == c)[0]
    u, v, w = F[f[oc], k[oc]], F[f[oc], (k[oc] + 1) % 3], F[f[oc], (k[oc] + 2) % 3]
    puv = V[u] + V[v]
    odd = F32(0.5) * puv
    if smooth:
        inner = count[oc] == 2
        odd[inner] = F32(0.375) * puv[inner] + F32(0.125) * (V[w[inner]] + V[other[oc[inner]]])
    Vn = np.empty((nv + E, 3), dtype=F32)
    Vn[:nv] = _loop_even(V, F, ok) if smooth else V
    Vn[nv + pos[oc]] = odd
    e = (nv + pos[own]).reshape(nf, 3)
    e01, e12, e20 = e[:, 0], e[:, 1], e[:, 2]
    Fn = np.stack([np.stack([F[:, 0], e01, e20], 1), np.stack([e01, F[:, 1], e12], 1), np.stack([e20, e12, F[:, 2]], 1),
                   np.stack([e01, e12, e20], 1)], 1).reshape(-1, 3)
    return Vn, Fn


def upsample(V, F, nr_subdivisions, smooth):
    """Mesh(V, F).upsample(nr_subdivisions, smooth) -> (V float32, F int32)"""
    V = np.array(V, dtype=F32).reshape(-1, 3)
    F = np.array(F, dtype=np.int64).reshape(-1, 3)
    for _ in range(nr_subdivisions):
        V, F = one_round(V, F, smooth)
    return V, F.astype(np.int32)
