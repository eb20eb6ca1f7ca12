"""Ray casting against a triangle mesh by brute force (numpy, fp32): the ray-triangle test of include/psdf_b200.h (two-sided
Moller-Trumbore, each operation rounded as written), tested against every triangle, and occluded / ambient_occlusion restated on top of it.
intersect also returns the test's t, u and v, for the first hits of tests/first_hit_oracle.py. csrc/mesh_raycast.cu gives the same answers
through its BVH."""
import math

import numpy as np

f32 = np.float32


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def intersect(p0, p1, p2, o, d, tnear, tfar):
    """the test of every pair of triangles (p0, p1, p2 [..., 3]) and rays (o, d [..., 3]), broadcast -> (pass bool [...], t, u, v float32
    [...]); t, u and v are meaningful where the test passes"""
    p0, p1, p2, o, d = (np.asarray(x, f32) for x in (p0, p1, p2, o, d))
    tnear, tfar = f32(tnear), f32(tfar)
    with np.errstate(all="ignore"):
        e1, e2 = p1 - p0, p2 - p0
        pv = cross(d, e2)
        det = dot(e1, pv)
        ok = (det != 0) & ~np.isnan(det)
        inv = f32(1) / det
        tv = o - p0
        u = dot(tv, pv) * inv
        ok &= (u >= 0) & (u <= 1)
        qv = cross(tv, e1)
        v = dot(d, qv) * inv
        ok &= (v >= 0) & (u + v <= 1)
        t = dot(e2, qv) * inv
        return ok & (t > tnear) & (t < tfar), t, u, v


def hit(p0, p1, p2, o, d, tnear, tfar):
    """the test of every pair of triangles (p0, p1, p2 [..., 3]) and rays (o, d [..., 3]), broadcast -> bool [...]"""
    return intersect(p0, p1, p2, o, d, tnear, tfar)[0]


def occluded(V, F, origins, dirs, tnear=1e-4, tfar=math.inf, chunk=1 << 22):
    """bool [R]: some triangle of (V [V,3], F [F,3]) passes the test for ray r"""
    V, F = np.asarray(V, f32), np.asarray(F, np.int64).reshape(-1, 3)
    o, d = np.asarray(origins, f32).reshape(-1, 3), np.asarray(dirs, f32).reshape(-1, 3)
    out = np.zeros(o.shape[0], bool)
    if F.shape[0] == 0:
        return out
    p0, p1, p2 = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    step = max(1, chunk // F.shape[0])
    for a in range(0, o.shape[0], step):
        out[a:a + step] = hit(p0[None], p1[None], p2[None], o[a:a + step, None], d[a:a + step, None], tnear, tfar).any(1)
    return out


def directions(S):
    """the fixed Fibonacci sphere of S directions: z = 1 - (2s + 1) / S, phi = s pi (3 - sqrt 5), r = sqrt(1 - z^2), (r cos phi, r sin phi,
    z), in fp64, rounded to fp32 -> [S,3]"""
    s = np.arange(S, dtype=np.float64)
    z = 1.0 - (2.0 * s + 1.0) / S
    phi = s * (math.pi * (3.0 - math.sqrt(5.0)))
    r = np.sqrt(np.maximum(0.0, 1.0 - z * z))
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1).astype(f32)


def ao_rays(V, NV, S):
    """the V S rays of ambient_occlusion, vertex-major -> (origins [V S,3], dirs [V S,3])"""
    V, NV = np.asarray(V, f32), np.asarray(NV, f32)
    D = directions(S)
    d = np.broadcast_to(D[None], (V.shape[0], S, 3))
    flip = dot(d, NV[:, None, :]) < 0
    d = np.where(flip[..., None], -d, d)
    o = np.broadcast_to(V[:, None, :], d.shape)
    return o.reshape(-1, 3), d.reshape(-1, 3)


def ambient_occlusion(V, F, NV, S):
    """vis [V] float32 = float(S - hits) / float(S) over the rays of ao_rays, tnear 1e-4, tfar inf"""
    o, d = ao_rays(V, NV, S)
    hits = occluded(V, F, o, d, f32(1e-4), math.inf).reshape(-1, S).sum(1)
    return ((S - hits).astype(f32) / f32(S)).astype(f32)
