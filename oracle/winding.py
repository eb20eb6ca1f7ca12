"""Generalized winding numbers by brute force in fp64 (numpy), the reference for csrc/mesh_winding.cu.

w(p) = (1/4 pi) sum over every face of its signed solid angle seen from p (Van Oosterom and Strackee 1983):
Omega = 2 atan2(det[a b c], |a||b||c| + (a.b)|c| + (b.c)|a| + (c.a)|b|), a, b, c = corners - p. A face contributes 0 when it repeats a
vertex, when its fp32 cross(p1 - p0, p2 - p0) is zero (equal or collinear corners), or when det == 0, as in the kernel, so winding_numbers is the exact sum that the kernel at beta = +inf rounds:
each of its terms is the fp32 form of the same formula, summed in fp64.

rounding_bound gives, per point, a bound on |kernel at beta = +inf - winding_numbers| from a first-order error analysis of that fp32
form (see its docstring). Points and faces are processed in chunks of about CHUNK point-face pairs, so 20 k faces x 100 k points stay
within a few hundred MB.
"""
import math

import numpy as np

CHUNK = 1 << 22
U32 = 2.0 ** -24


def _gamma(n):
    return n * U32 / (1 - n * U32)


def zero_area(tri32):
    """[F] bool: cross(p1 - p0, p2 - p0) == 0 in fp32, rounded as the kernel rounds it (equal or collinear corners)"""
    e1, e2 = tri32[:, 1] - tri32[:, 0], tri32[:, 2] - tri32[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    return np.all(n == 0, axis=1)


def _corners(verts, faces):
    """fp64 corners [F,3,3] of the faces that contribute: not repeating a vertex and not of zero fp32 area"""
    V = np.asarray(verts, np.float32)
    Fi = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(Fi) == 0:
        return np.zeros((0, 3, 3))
    tri = V[Fi]
    rep = (Fi[:, 0] == Fi[:, 1]) | (Fi[:, 1] == Fi[:, 2]) | (Fi[:, 2] == Fi[:, 0])
    return tri[~(rep | zero_area(tri))].astype(np.float64)


def _terms(points, tri):
    """per (point, face) of a chunk: y = det, x = den in fp64 and the componentwise magnitudes Dy, Dx that bound their fp32 rounding"""
    a = tri[None, :, 0, :] - points[:, None, :]
    b = tri[None, :, 1, :] - points[:, None, :]
    c = tri[None, :, 2, :] - points[:, None, :]
    bc = np.cross(b, c)
    y = np.einsum("pfk,pfk->pf", a, bc)
    la, lb, lc = (np.sqrt(np.einsum("pfk,pfk->pf", v, v)) for v in (a, b, c))
    ab, bcd, ca = (np.einsum("pfk,pfk->pf", u, v) for u, v in ((a, b), (b, c), (c, a)))
    x = la * lb * lc + ab * lc + bcd * la + ca * lb
    A, B, C = np.abs(a), np.abs(b), np.abs(c)
    Dy = np.einsum("pfk,pfk->pf", A, B[..., [1, 2, 0]] * C[..., [2, 0, 1]] + B[..., [2, 0, 1]] * C[..., [1, 2, 0]])
    Dx = la * lb * lc + np.einsum("pfk,pfk->pf", A, B) * lc + np.einsum("pfk,pfk->pf", B, C) * la + np.einsum("pfk,pfk->pf", C, A) * lb
    return y, x, Dy, Dx


def _chunks(P, F):
    step = max(1, CHUNK // max(F, 1))
    return range(0, P, step), step


def winding_numbers(verts, faces, points):
    """fp64 [P]: (1/4 pi) sum over the contributing faces of 2 atan2(det, den), the faces in index order"""
    tri = _corners(verts, faces)
    p = np.asarray(points, np.float32).astype(np.float64).reshape(-1, 3)
    out = np.zeros(len(p))
    if len(tri) == 0:
        return out
    starts, step = _chunks(len(p), len(tri))
    for s in starts:
        y, x, _, _ = _terms(p[s:s + step], tri)
        om = np.where(y != 0, 2.0 * np.arctan2(y, x), 0.0)
        out[s:s + step] = om.sum(axis=1) / (4 * math.pi)
    return out


def rounding_bound(verts, faces, points):
    """fp64 [P]: a bound on |w32 - winding_numbers| for w32 the kernel's exact (beta = +inf) value, whose terms are the fp32 form of the
    solid angle. Per face, with u = 2^-24 and gamma_n = n u / (1 - n u):
      the fp32 det (corner differences, cross, dot) is within dy = gamma_12 Dy of y, Dy = sum over the six products |a_i b_j c_k|;
      the fp32 den (three lengths, three dots, products and sums) is within dx = gamma_20 Dx of x, Dx = |a||b||c| + sum|a_i b_i| |c| + ...
      Dy == 0: every product is 0, both forms give y = 0 and skip the face: 0.
      x > dx or |y| > dy: atan2 is smooth on the box of (y, x) values, so the angle moves by at most (dx + dy) / (|(y, x)| - dx - dy)
        (pi when that distance is not positive); else the sign of y or x is undecided and the angle can be anything: 2 pi.
      atan2f adds at most 4 ulp of its result (2^-21 |theta| + 2^-149).
    Omega = 2 theta, so each face contributes 2 (that bound, at most 2 pi) / 4 pi; plus the fp64 sum of F terms (gamma_F of fp64 times
    sum |Omega| / 4 pi) and the final rounding to fp32 (2^-24 |w| + 2^-149)."""
    tri = _corners(verts, faces)
    p = np.asarray(points, np.float32).astype(np.float64).reshape(-1, 3)
    out = np.zeros(len(p))
    if len(tri) == 0:
        return out
    F = len(tri)
    starts, step = _chunks(len(p), F)
    g64 = F * 2.0 ** -53 / (1 - F * 2.0 ** -53)
    for s in starts:
        y, x, Dy, Dx = _terms(p[s:s + step], tri)
        dy, dx = _gamma(12) * Dy, _gamma(20) * Dx
        gap = np.hypot(x, y) - dx - dy
        with np.errstate(divide="ignore", invalid="ignore"):
            smooth = np.where(gap > 0, (dx + dy) / gap, math.pi)
        theta = np.where((x > dx) | (np.abs(y) > dy), np.minimum(smooth, 2 * math.pi), 2 * math.pi)
        theta = np.where(Dy == 0, 0.0, theta + 2.0 ** -21 * np.abs(np.arctan2(y, x)) + 2.0 ** -149)
        om = np.where(y != 0, 2.0 * np.arctan2(y, x), 0.0)
        w = om.sum(axis=1) / (4 * math.pi)
        out[s:s + step] = (2 * theta).sum(axis=1) / (4 * math.pi) + g64 * np.abs(om).sum(axis=1) / (4 * math.pi) + 2.0 ** -24 * np.abs(w) + 2.0 ** -149
    return out
