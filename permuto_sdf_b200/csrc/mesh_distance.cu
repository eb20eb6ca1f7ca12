// Closest points on an indexed triangle mesh through the BVH of mesh_bvh.cu, angle-weighted pseudonormals, signed distances and
// area-weighted surface samples, sm_90a. Built with -fmad=false: the closest-point formula is rounded operation by operation as
// include/psdf_b200.h states it, so oracle/mesh_distance.py (brute force over all faces) reproduces dist2, face and bary bit for bit.
// The tree only prunes: a node is skipped when the fp32 distance to its padded box is strictly above the best squared distance so far,
// and that bound never exceeds the computed distance of a face inside (see the header). The pseudonormals sum over the vertex -> face
// CSR of mesh_csr.cuh.
//
//   k_md_closest   dist2, face, bary of the nearest valid face, traverse of mesh_bvh.cuh             thread per point
//   k_md_sign      sign of dot(p - q, pseudonormal of the closest feature) times sqrt(dist2)         thread per point
//   k_md_face_n    unit face normal                                                                  thread per face
//   k_md_vert_n    sum of angle * face normal over the vertex's faces, ascending                     thread per vertex
//   k_md_edge_n    sum of the face normals of the faces holding both ends of a face edge, ascending  thread per (face, corner)
//   k_md_sample    area-weighted sample k from SplitMix64 outputs 3k + 1 .. 3k + 3                    thread per sample
#include "mesh_bvh.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
// ---------------------------------------------------------------- closest point on a triangle (include/psdf_b200.h)
struct Closest {
    float d2;
    float b0, b1, b2;
};

__device__ __forceinline__ float dist2(float3 p, float3 q) {
    const float3 d = sub3(p, q);
    return dot3(d, d);
}

// x + t e, per coordinate
__device__ __forceinline__ float3 along(float3 x, float3 e, float t) { return make_float3(x.x + t * e.x, x.y + t * e.y, x.z + t * e.z); }

// the clamped projection of p on segment x -> y: t = dot(p - x, e) / dot(e, e) (0 when dot(e, e) is 0), clamped to [0, 1]
__device__ __forceinline__ float segment_t(float3 p, float3 x, float3 e) {
    const float ee = dot3(e, e);
    const float t = ee > 0.0f ? dot3(sub3(p, x), e) / ee : 0.0f;
    return fminf(fmaxf(t, 0.0f), 1.0f);
}

// the nearest of the edges ab, bc, ca (a strictly smaller dist2 wins): zero-area faces and the interior fallback
__device__ Closest nearest_edge(float3 p, float3 a, float3 b, float3 c) {
    const float3 ab = sub3(b, a), bc = sub3(c, b), ca = sub3(a, c);
    const float t0 = segment_t(p, a, ab), t1 = segment_t(p, b, bc), t2 = segment_t(p, c, ca);
    Closest r{dist2(p, along(a, ab, t0)), 1.0f - t0, t0, 0.0f};
    const float d1 = dist2(p, along(b, bc, t1));
    if (d1 < r.d2) r = Closest{d1, 0.0f, 1.0f - t1, t1};
    const float d2 = dist2(p, along(c, ca, t2));
    if (d2 < r.d2) r = Closest{d2, t2, 0.0f, 1.0f - t2};
    return r;
}

// Ericson's region test (Real-Time Collision Detection, 5.1.5) with every division guarded. The signed areas va, vb, vc are the
// book's triple products rather than its d1 d4 - d3 d2 products: those cancel to nothing on a sliver (|n|^2 far below the rounding of
// |ab|^2 |ap|^2) and send points inside it to an edge or a corner, while the triple products keep a relative error of about eps |e| / h.
__device__ Closest closest_on_triangle(float3 p, float3 a, float3 b, float3 c) {
    const float3 ab = sub3(b, a), ac = sub3(c, a);
    const float3 n = cross3(ab, ac);
    if (n.x == 0.0f && n.y == 0.0f && n.z == 0.0f) return nearest_edge(p, a, b, c);
    const float3 ap = sub3(p, a);
    const float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) return Closest{dist2(p, a), 1.0f, 0.0f, 0.0f};
    const float3 bp = sub3(p, b);
    const float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) return Closest{dist2(p, b), 0.0f, 1.0f, 0.0f};
    const float vc = dot3(n, cross3(ap, bp));
    const float eab = d1 - d3;
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f && eab > 0.0f) {
        const float v = d1 / eab;
        return Closest{dist2(p, along(a, ab, v)), 1.0f - v, v, 0.0f};
    }
    const float3 cp = sub3(p, c);
    const float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) return Closest{dist2(p, c), 0.0f, 0.0f, 1.0f};
    const float vb = dot3(n, cross3(cp, ap));
    const float eac = d2 - d6;
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f && eac > 0.0f) {
        const float w = d2 / eac;
        return Closest{dist2(p, along(a, ac, w)), 1.0f - w, 0.0f, w};
    }
    const float va = dot3(n, cross3(bp, cp));
    const float e43 = d4 - d3, e56 = d5 - d6;
    const float ebc = e43 + e56;
    if (va <= 0.0f && e43 >= 0.0f && e56 >= 0.0f && ebc > 0.0f) {
        const float w = e43 / ebc;
        return Closest{dist2(p, along(b, sub3(c, b), w)), 0.0f, 1.0f - w, w};
    }
    const float den = (va + vb) + vc;
    if (den > 0.0f) {
        const float v = vb / den, w = vc / den;
        if (v >= 0.0f && w >= 0.0f && v + w <= 1.0f) {             // the nearest edge when it is closer: a sliver's weights are
            const Closest e = nearest_edge(p, a, b, c);             // too coarse to place q within its width
            const float d = dist2(p, along(along(a, ab, v), ac, w));
            return e.d2 < d ? e : Closest{d, (1.0f - v) - w, v, w};
        }
    }
    return nearest_edge(p, a, b, c);
}

// ---------------------------------------------------------------- traversal
// squared fp32 distance from p to the box grown by pad: per axis max(lo - pad - p, p - (hi + pad), 0), summed as dot3
__device__ __forceinline__ float box_d2(const Box& b, float3 p, float pad) {
    const float ex = fmaxf(fmaxf((b.lo.x - pad) - p.x, p.x - (b.hi.x + pad)), 0.0f);
    const float ey = fmaxf(fmaxf((b.lo.y - pad) - p.y, p.y - (b.hi.y + pad)), 0.0f);
    const float ez = fmaxf(fmaxf((b.lo.z - pad) - p.z, p.z - (b.hi.z + pad)), 0.0f);
    return (ex * ex + ey * ey) + ez * ez;
}

struct Best {
    float d2;
    int face;
    float b0, b1, b2;
};

// sorted leaf i: taken when its dist2 is smaller, or equal with a smaller original face; faces that repeat a vertex are skipped
__device__ __forceinline__ void visit_leaf(const Ws& W, const int* __restrict__ faces, long long i, float3 p, Best& best) {
    float3 a, b, c;
    leaf_corners(W, i, a, b, c);
    const Closest r = closest_on_triangle(p, a, b, c);
    if (!(r.d2 <= best.d2)) return;                           // also NaN: the corners of a face refused by the caller
    const int f = __ldg(W.vals0 + i);
    if (!(r.d2 < best.d2 || f < best.face)) return;
    if (!distinct(load_face(faces, f))) return;
    best = Best{r.d2, f, r.b0, r.b1, r.b2};
}

// the nearest face (traverse): the key is the box bound, and a box is kept while its bound is not above the best dist2, so ties are visited
struct Nearest {
    const Ws& W;
    const int* __restrict__ faces;
    float3 p;
    float pad;
    Best best;
    __device__ bool keep(float key) const { return key <= best.d2; }
    __device__ bool enter(const Box& b, float& key) const {
        key = box_d2(b, p, pad);
        return keep(key);
    }
    __device__ bool visit(long long i) {
        visit_leaf(W, faces, i, p, best);
        return false;
    }
};

__device__ Best nearest(const Ws& W, const int* __restrict__ faces, int F, float3 p, float pad) {
    Nearest q{W, faces, p, pad, Best{INFINITY, -1, 0.0f, 0.0f, 0.0f}};
    traverse(W, F, q);
    return q.best;
}

__global__ void __launch_bounds__(kThreads) k_md_closest(int F, long long P, const float* __restrict__ points, const int* __restrict__ faces,
                                                         Ws W, float* __restrict__ dist2_out, int* __restrict__ face_out,
                                                         float* __restrict__ bary_out) {
    const long long i = thread_index();
    if (i >= P) return;
    const Best r = nearest(W, faces, F, load3(points, i), kPad * mesh_scale(W));
    dist2_out[i] = r.d2;
    face_out[i] = r.face;
    bary_out[3 * i] = r.b0;
    bary_out[3 * i + 1] = r.b1;
    bary_out[3 * i + 2] = r.b2;
}

// the pseudonormal of the feature the barycentrics name: two zero weights a vertex, one an edge, none the face
__device__ __forceinline__ float3 feature_normal(long long f, int3 t, float b0, float b1, float b2, const float* __restrict__ face_n,
                                                 const float* __restrict__ vert_n, const float* __restrict__ edge_n) {
    const int zeros = (b0 == 0.0f) + (b1 == 0.0f) + (b2 == 0.0f);
    if (zeros == 2) return load3(vert_n, b0 != 0.0f ? t.x : (b1 != 0.0f ? t.y : t.z));
    if (zeros == 1) return load3(edge_n, 3 * f + (b2 == 0.0f ? 0 : (b0 == 0.0f ? 1 : 2)));
    return load3(face_n, f);
}

__global__ void __launch_bounds__(kThreads) k_md_sign(long long P, const float* __restrict__ points, const float* __restrict__ verts,
                                                      const int* __restrict__ faces, const float* __restrict__ face_n,
                                                      const float* __restrict__ vert_n, const float* __restrict__ edge_n,
                                                      const float* __restrict__ dist2, const int* __restrict__ face,
                                                      const float* __restrict__ bary, float* __restrict__ sdf) {
    const long long i = thread_index();
    if (i >= P) return;
    const int f = face[i];
    const float d = sqrtf(dist2[i]);
    if (f < 0) {
        sdf[i] = d;                                           // no valid face: +inf
        return;
    }
    const int3 t = load_face(faces, f);
    const float b0 = bary[3 * i], b1 = bary[3 * i + 1], b2 = bary[3 * i + 2];
    const float3 a = load3(verts, t.x), b = load3(verts, t.y), c = load3(verts, t.z);
    const float3 q = make_float3((b0 * a.x + b1 * b.x) + b2 * c.x, (b0 * a.y + b1 * b.y) + b2 * c.y, (b0 * a.z + b1 * b.z) + b2 * c.z);
    const float s = dot3(sub3(load3(points, i), q), feature_normal(f, t, b0, b1, b2, face_n, vert_n, edge_n));
    sdf[i] = s > 0.0f ? d : (s < 0.0f ? -d : 0.0f);
}

// ---------------------------------------------------------------- pseudonormals
struct PnWs {
    long long* info;          // {faces outside [0, V), faces repeating a vertex, 0, 0}
    long long* off;           // [V + 1] CSR offsets
    int* deg;                 // [V] face count, then the fill cursor
    int* adj;                 // [3F] faces of each vertex, ascending
    long long* tiles;         // scan tile sums
};

long long carve_pn(void* ws, long long V, long long F, PnWs* W) {
    Sections s{static_cast<char*>(ws)};
    PnWs w;
    s.take(w.info, kHeaderBytes);
    s.take(w.off, 8 * (V + 1));
    s.take(w.deg, 4 * V);
    s.take(w.adj, 12 * F);
    s.take(w.tiles, 8 * tile_sums(V));
    if (W) *W = w;
    return s.size;
}

__device__ __forceinline__ void store3(float* __restrict__ out, long long i, float3 v) {
    out[3 * i] = v.x;
    out[3 * i + 1] = v.y;
    out[3 * i + 2] = v.z;
}

__global__ void __launch_bounds__(kThreads) k_md_face_n(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces,
                                                        float* __restrict__ face_n) {
    const long long f = thread_index();
    if (f >= F) return;
    const int3 t = load_face(faces, f);
    float3 n = make_float3(0.0f, 0.0f, 0.0f);
    if (valid(t, V)) {
        const float3 a = load3(verts, t.x);
        n = cross3(sub3(load3(verts, t.y), a), sub3(load3(verts, t.z), a));
        const float l = sqrtf(dot3(n, n));
        n = l > 0.0f ? make_float3(n.x / l, n.y / l, n.z / l) : make_float3(0.0f, 0.0f, 0.0f);
    }
    store3(face_n, f, n);
}

__global__ void __launch_bounds__(kThreads) k_md_vert_n(int V, const float* __restrict__ verts, const int* __restrict__ faces,
                                                        const float* __restrict__ face_n, PnWs W, float* __restrict__ vert_n) {
    const long long v = thread_index();
    if (v >= V) return;
    const float3 p = load3(verts, v);
    float3 s = make_float3(0.0f, 0.0f, 0.0f);
    for (long long i = W.off[v], e = W.off[v + 1]; i < e; i++) {
        const int f = W.adj[i];
        const int3 t = load_face(faces, f);
        const int k = t.x == v ? 0 : (t.y == v ? 1 : 2);
        const float3 e1 = sub3(load3(verts, corner(t, (k + 1) % 3)), p), e2 = sub3(load3(verts, corner(t, (k + 2) % 3)), p);
        const float3 c = cross3(e1, e2);
        const float angle = atan2f(sqrtf(dot3(c, c)), dot3(e1, e2));
        const float3 n = load3(face_n, f);
        s = make_float3(s.x + angle * n.x, s.y + angle * n.y, s.z + angle * n.z);
    }
    store3(vert_n, v, s);
}

__global__ void __launch_bounds__(kThreads) k_md_edge_n(int V, int F, const int* __restrict__ faces, const float* __restrict__ face_n, PnWs W,
                                                        float* __restrict__ edge_n) {
    const long long e = thread_index();
    if (e >= 3LL * F) return;
    const long long f = e / 3;
    const int k = (int)(e - 3 * f);
    const int3 t = load_face(faces, f);
    float3 s = make_float3(0.0f, 0.0f, 0.0f);
    if (valid(t, V)) {
        const int u = corner(t, k), v = corner(t, (k + 1) % 3);
        const int w = nr_faces(W, u) <= nr_faces(W, v) ? u : v;    // both lists are ascending: the shorter one gives the same sum
        const int o = w == u ? v : u;
        for (long long i = W.off[w], end = W.off[w + 1]; i < end; i++) {
            const int g = W.adj[i];
            const int3 tg = load_face(faces, g);
            if (tg.x == o || tg.y == o || tg.z == o) {
                const float3 n = load3(face_n, g);
                s = make_float3(s.x + n.x, s.y + n.y, s.z + n.z);
            }
        }
    }
    store3(edge_n, e, s);
}

// ---------------------------------------------------------------- surface samples
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long seed, unsigned long long n) {
    unsigned long long z = seed + (n + 1) * 0x9E3779B97F4A7C15ull;     // output n of SplitMix64 seeded with seed
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__global__ void __launch_bounds__(kThreads) k_md_sample(int F, const float* __restrict__ verts, const int* __restrict__ faces,
                                                        const double* __restrict__ cdf, long long N, unsigned long long seed,
                                                        float* __restrict__ points_out, int* __restrict__ face_out) {
    const long long k = thread_index();
    if (k >= N) return;
    const unsigned long long n = 3ull * (unsigned long long)k;
    const double total = cdf[F - 1];
    const double u0 = (double)(splitmix64(seed, n) >> 11) * 0x1p-53 * total;
    const bool top = !(u0 < total);                            // u0 rounded up to the total: the first face that reaches it
    int lo = 0, hi = F - 1;
    while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        if (top ? cdf[mid] >= total : cdf[mid] > u0) hi = mid;
        else lo = mid + 1;
    }
    const float r1 = (float)(splitmix64(seed, n + 1) >> 40) * 0x1p-24f, r2 = (float)(splitmix64(seed, n + 2) >> 40) * 0x1p-24f;
    const float s = sqrtf(r1);
    const float b0 = 1.0f - s, b1 = s * (1.0f - r2), b2 = s * r2;
    const int3 t = load_face(faces, lo);
    const float3 a = load3(verts, t.x), b = load3(verts, t.y), c = load3(verts, t.z);
    store3(points_out, k, make_float3((b0 * a.x + b1 * b.x) + b2 * c.x, (b0 * a.y + b1 * b.y) + b2 * c.y, (b0 * a.z + b1 * b.z) + b2 * c.z));
    face_out[k] = lo;
}
}  // namespace

extern "C" {

int psdf_mesh_closest_points(int V, int F, long long P, const float* points, const float* verts, const int* faces, const uint8_t* workspace,
                             float* dist2_out, int* face_out, float* bary_out, void* stream) {
    if (V < 0 || F < 0 || P < 0 || !workspace || (F > 0 && !faces) || (P > 0 && (!points || !dist2_out || !face_out || !bary_out)))
        return PSDF_ERR_ARG;
    if (P > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    (void)verts;
    if (P == 0) return PSDF_OK;
    Ws W;
    carve(const_cast<uint8_t*>(workspace), V, F, &W);
    k_md_closest<<<blocks(P), kThreads, 0, ST>>>(F, P, points, faces, W, dist2_out, face_out, bary_out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

long long psdf_mesh_pseudonormals_workspace_bytes(long long nr_vertices, long long nr_faces) {
    if (nr_vertices < 0 || nr_faces < 0) return PSDF_ERR_ARG;
    if (nr_vertices > kIntMax || nr_faces > kIntMax) return PSDF_ERR_UNSUPPORTED;
    return carve_pn(nullptr, nr_vertices, nr_faces, nullptr);
}

int psdf_mesh_pseudonormals(int V, int F, const float* verts, const int* faces, uint8_t* workspace, float* face_n, float* vert_n,
                            float* edge_n, void* stream) {
    if (V < 0 || F < 0 || !workspace || (V > 0 && (!verts || !vert_n)) || (F > 0 && (!faces || !face_n || !edge_n))) return PSDF_ERR_ARG;
    PnWs W;
    carve_pn(workspace, V, F, &W);
    cudaMemsetAsync(W.info, 0, kHeaderBytes, ST);
    if (F > 0) k_mesh_check<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
    build_csr(V, F, faces, W, true, ST);
    if (F > 0) k_md_face_n<<<blocks(F), kThreads, 0, ST>>>(V, F, verts, faces, face_n);
    if (V > 0) k_md_vert_n<<<blocks(V), kThreads, 0, ST>>>(V, verts, faces, face_n, W, vert_n);
    if (F > 0) k_md_edge_n<<<blocks(3LL * F), kThreads, 0, ST>>>(V, F, faces, face_n, W, edge_n);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_signed_distance(int V, int F, long long P, const float* points, const float* verts, const int* faces, const uint8_t* workspace,
                              const float* face_n, const float* vert_n, const float* edge_n, float* dist2_out, int* face_out,
                              float* bary_out, float* sdf_out, void* stream) {
    if (V < 0 || F < 0 || P < 0 || !workspace || (F > 0 && (!faces || !verts || !face_n || !vert_n || !edge_n)) ||
        (P > 0 && (!points || !dist2_out || !face_out || !bary_out || !sdf_out)))
        return PSDF_ERR_ARG;
    if (P > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    if (P == 0) return PSDF_OK;
    Ws W;
    carve(const_cast<uint8_t*>(workspace), V, F, &W);
    k_md_closest<<<blocks(P), kThreads, 0, ST>>>(F, P, points, faces, W, dist2_out, face_out, bary_out);
    k_md_sign<<<blocks(P), kThreads, 0, ST>>>(P, points, verts, faces, face_n, vert_n, edge_n, dist2_out, face_out, bary_out, sdf_out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_sample_surface(int V, int F, const float* verts, const int* faces, const double* cdf, long long N, uint64_t seed,
                             float* points_out, int* face_out, void* stream) {
    if (V < 0 || F < 0 || N < 0 || (N > 0 && (F == 0 || !verts || !faces || !cdf || !points_out || !face_out))) return PSDF_ERR_ARG;
    if (N > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    if (N == 0) return PSDF_OK;
    k_md_sample<<<blocks(N), kThreads, 0, ST>>>(F, verts, faces, cdf, N, seed, points_out, face_out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
