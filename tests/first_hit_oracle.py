"""The first-hit answer of psdf_mesh_first_hit and the per-pixel shading of psdf_mesh_render, by brute force in numpy fp32 (test
infrastructure): the ray-triangle test of include/psdf_b200.h (oracle/raycast.py's intersect, each operation rounded as written, with its
t, u and v) against every triangle. csrc/mesh_raycast.cu gives the same answers through its BVH."""
import math

import numpy as np

from oracle.raycast import cross, dot, intersect

f32 = np.float32


def first_hit(V, F, origins, dirs, tnear=0.0, tfar=math.inf, chunk=1 << 22):
    """psdf_mesh_first_hit by brute force -> (t float32 [R], face int32 [R], bary float32 [R,3]): of the faces that pass the test, the
    smallest t, ties to the smallest face index; bary = ((1 - u) - v, u, v). No such face: (+inf, -1, 0)."""
    V, F = np.asarray(V, f32), np.asarray(F, np.int64).reshape(-1, 3)
    o, d = np.asarray(origins, f32).reshape(-1, 3), np.asarray(dirs, f32).reshape(-1, 3)
    R = o.shape[0]
    t_out = np.full(R, np.inf, f32)
    face = np.full(R, -1, np.int32)
    bary = np.zeros((R, 3), f32)
    if F.shape[0] == 0:
        return t_out, face, bary
    p0, p1, p2 = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    step = max(1, chunk // F.shape[0])
    for a in range(0, R, step):
        ok, t, u, v = intersect(p0[None], p1[None], p2[None], o[a:a + step, None], d[a:a + step, None], tnear, tfar)
        t = np.where(ok, t, f32(np.inf))
        tmin = t.min(1)
        rows = np.flatnonzero(ok.any(1))
        first = np.argmax(ok & (t == tmin[:, None]), 1)[rows]           # the smallest face index among the ties
        r = rows + a
        uu, vv = u[rows, first], v[rows, first]
        t_out[r], face[r] = tmin[rows], first
        bary[r] = np.stack([(f32(1) - uu) - vv, uu, vv], 1)
    return t_out, face, bary


def shade(V, F, t, face, bary, normals=None, colors=None):
    """the per-pixel outputs of psdf_mesh_render from first hits (t, face, bary as first_hit gives them) -> dict of rgb [R,3], mask [R],
    depth [R], normal [R,3] (float32) and face [R] (int32): on a hit of face (a, b, c), n = (b0 N_a + b1 N_b) + b2 N_c with normals,
    else cross(p_b - p_a, p_c - p_a); l = sqrt(dot(n, n)), n = n / l (0 when l == 0); rgb = (b0 C_a + b1 C_b) + b2 C_c with colors, else
    0.5 + 0.5 n; mask 1, depth t. A miss: all 0 and face -1."""
    V, F = np.asarray(V, f32), np.asarray(F, np.int64).reshape(-1, 3)
    t, face, bary = np.asarray(t, f32), np.asarray(face, np.int32), np.asarray(bary, f32)
    R = face.shape[0]
    rgb, normal = np.zeros((R, 3), f32), np.zeros((R, 3), f32)
    mask, depth = np.zeros(R, f32), np.zeros(R, f32)
    h = np.flatnonzero(face >= 0)
    tri = F[face[h]]
    b0, b1, b2 = (bary[h, k:k + 1] for k in range(3))

    def blend(A):
        A = np.asarray(A, f32)
        return (b0 * A[tri[:, 0]] + b1 * A[tri[:, 1]]) + b2 * A[tri[:, 2]]

    if normals is not None:
        n = blend(normals)
    else:
        n = cross(V[tri[:, 1]] - V[tri[:, 0]], V[tri[:, 2]] - V[tri[:, 0]])
    l = np.sqrt(dot(n, n))[:, None]
    with np.errstate(all="ignore"):
        n = np.where(l == 0, f32(0), n / l).astype(f32)
    rgb[h] = blend(colors) if colors is not None else f32(0.5) + f32(0.5) * n
    normal[h], mask[h], depth[h] = n, 1, t[h]
    return {"rgb": rgb, "mask": mask, "depth": depth, "normal": normal, "face": face.copy()}
