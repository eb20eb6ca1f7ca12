// Any-hit and first-hit ray casting against an indexed triangle mesh through a linear BVH, per-vertex ambient occlusion and rendering from
// reel cameras, sm_90a. Built with -fmad=false: the ray-triangle test is rounded operation by operation as include/psdf_b200.h states it,
// so oracle/raycast.py and, for first hits, tests/first_hit_oracle.py (brute force over all triangles) reproduce every answer. The tree
// only decides which triangles are tested; the answer is "some triangle passes", or for first hits the passing triangle of smallest t,
// ties to the smallest original face index.
//
// Build (psdf_mesh_bvh_build): the centroids' bounds and the largest |coordinate| are reduced with ordered-key atomics (k_rc_bounds);
// each face gets the 30-bit Morton code of its centroid within those bounds (k_rc_morton); four stable 8-bit LSD radix passes
// (k_rc_hist, the int64 scan of mesh_csr.cuh over the digit-major tile histogram, k_rc_scatter) sort the faces by code; Karras' radix
// tree over the sorted codes, ties broken by sorted position, gives the F - 1 internal nodes (k_rc_internal); k_rc_leaves writes each
// leaf's triangle in sorted order and refits the boxes bottom-up, the second child to arrive at a node going on.
//
//   k_rc_bounds     centroid bounds and max |coordinate| of the valid faces                          thread per face
//   k_rc_morton     Morton code and face index                                                      thread per face
//   k_rc_hist       per-tile counts of one 8-bit digit, digit-major                                 tile of 256 faces
//   k_rc_scatter    stable scatter of one digit                                                     tile of 256 faces
//   k_rc_internal   children and parents of internal node i (Karras 2012)                            thread per internal node
//   k_rc_leaves     leaf triangles and the bottom-up box refit                                       thread per leaf
//   k_rc_occluded   hit_out[r] = any hit of ray r                                                    thread per ray
//   k_fh_rays       t, face, bary of the first hit of ray r, nearer child first                      thread per ray
//   k_fh_render     first hit of the reel ray of each pixel, shaded into NCHW images                 thread per (image, pixel), warp per 8 x 4 tile
//   k_rc_ao         hits[i] += any hit of (V[i], dirs[s] flipped to NV[i]'s side)                    thread per (vertex, direction)
//   k_rc_vis        vis[i] = float(S - hits[i]) / float(S)                                           thread per vertex
#include "mesh_bvh.cuh"
#include "reel_ray.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr int kWarps = kThreads / 32;
constexpr float kSlabRel = 1.0f / 1048576.0f;   // relative slack of the slab test's far end: above 2 gamma_3 of fp32 (Ize 2013)

// two-sided Moller-Trumbore as include/psdf_b200.h states it; on a pass, t, u and v as computed
__device__ __forceinline__ bool hit_triangle(float3 p0, float3 p1, float3 p2, float3 o, float3 d, float tnear, float tfar, float& t, float& u,
                                             float& v) {
    const float3 e1 = sub3(p1, p0), e2 = sub3(p2, p0);
    const float3 pv = cross3(d, e2);
    const float det = dot3(e1, pv);
    if (det == 0.0f || det != det) return false;
    const float inv = 1.0f / det;
    const float3 tv = sub3(o, p0);
    u = dot3(tv, pv) * inv;
    if (!(u >= 0.0f && u <= 1.0f)) return false;
    const float3 qv = cross3(tv, e1);
    v = dot3(d, qv) * inv;
    if (!(v >= 0.0f && u + v <= 1.0f)) return false;
    t = dot3(e2, qv) * inv;
    return t > tnear && t < tfar;
}

__device__ __forceinline__ unsigned float_key(float f) {
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__device__ __forceinline__ float3 centroid(float3 a, float3 b, float3 c) {
    const float k = 1.0f / 3.0f;
    return make_float3(((a.x + b.x) + c.x) * k, ((a.y + b.y) + c.y) * k, ((a.z + b.z) + c.z) * k);
}

// ---------------------------------------------------------------- build
__global__ void __launch_bounds__(kThreads) k_rc_bounds(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u}, amax = 0u;
    if (f < F) {
        const int3 t = load_face(faces, f);
        if (in_range(t, V)) {
            const float3 a = load3(verts, t.x), b = load3(verts, t.y), c = load3(verts, t.z);
            const float3 m = centroid(a, b, c);
            lo[0] = hi[0] = float_key(m.x);
            lo[1] = hi[1] = float_key(m.y);
            lo[2] = hi[2] = float_key(m.z);
            const float x = fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(b.x))),
                                  fmaxf(fmaxf(fabsf(b.y), fabsf(b.z)), fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fabsf(c.z))));
            amax = __float_as_uint(x);                // non-negative floats order as their bits
        }
    }
    for (int k = 0; k < 3; k++) {
        lo[k] = __reduce_min_sync(kFullMask, lo[k]);
        hi[k] = __reduce_max_sync(kFullMask, hi[k]);
    }
    amax = __reduce_max_sync(kFullMask, amax);
    if ((threadIdx.x & 31) == 0) {
        for (int k = 0; k < 3; k++) {
            if (lo[k] != 0xffffffffu) atomicMin(W.bounds + k, lo[k]);
            if (hi[k]) atomicMax(W.bounds + 3 + k, hi[k]);
        }
        if (amax) atomicMax(W.bounds + 6, amax);
    }
}

__device__ __forceinline__ unsigned spread10(unsigned x) {       // 10 bits -> every third bit
    x = (x | (x << 16)) & 0x030000ffu;
    x = (x | (x << 8)) & 0x0300f00fu;
    x = (x | (x << 4)) & 0x030c30c3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}

__device__ __forceinline__ unsigned quantize(float c, float lo, float hi) {
    const float e = hi - lo;
    const float q = e > 0.0f ? (c - lo) / e * 1024.0f : 0.0f;
    return (unsigned)fminf(fmaxf(q, 0.0f), 1023.0f);
}

__global__ void __launch_bounds__(kThreads) k_rc_morton(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    if (f >= F) return;
    const int3 t = load_face(faces, f);
    unsigned code = 0;
    if (in_range(t, V)) {
        const float3 m = centroid(load3(verts, t.x), load3(verts, t.y), load3(verts, t.z));
        float lo[3], hi[3];
        for (int k = 0; k < 3; k++) {
            lo[k] = key_float(W.bounds[k]);
            hi[k] = key_float(W.bounds[3 + k]);
        }
        code = (spread10(quantize(m.x, lo[0], hi[0])) << 2) | (spread10(quantize(m.y, lo[1], hi[1])) << 1) |
               spread10(quantize(m.z, lo[2], hi[2]));
    }
    W.keys0[f] = code;
    W.vals0[f] = (int)f;
}

__global__ void __launch_bounds__(kThreads) k_rc_hist(int F, const unsigned* __restrict__ keys, int shift, int* __restrict__ hist,
                                                      long long ntiles) {
    __shared__ int cnt[kDigits];
    const long long i = thread_index();
    cnt[threadIdx.x] = 0;
    __syncthreads();
    if (i < F) atomicAdd(cnt + ((keys[i] >> shift) & 255u), 1);
    __syncthreads();
    hist[(long long)threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
}

// stable within a tile: ranks follow thread order (warp by warp, lane by lane); across tiles the digit-major prefix keeps tile order
__global__ void __launch_bounds__(kThreads) k_rc_scatter(int F, const unsigned* __restrict__ keys, const int* __restrict__ vals, int shift,
                                                         const long long* __restrict__ off, long long ntiles, unsigned* __restrict__ keys_out,
                                                         int* __restrict__ vals_out) {
    __shared__ int wc[kWarps][kDigits];
    const long long i = thread_index();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int w = 0; w < kWarps; w++) wc[w][threadIdx.x] = 0;
    __syncthreads();
    const bool ok = i < F;
    const unsigned key = ok ? keys[i] : 0u;
    const int digit = ok ? (int)((key >> shift) & 255u) : kDigits;
    const unsigned peers = __match_any_sync(kFullMask, digit);
    const unsigned below = peers & ((1u << lane) - 1u);
    if (ok && !below) wc[warp][digit] = __popc(peers);
    __syncthreads();
    int s = 0;
    for (int w = 0; w < kWarps; w++) {
        const int c = wc[w][threadIdx.x];
        wc[w][threadIdx.x] = s;
        s += c;
    }
    __syncthreads();
    if (!ok) return;
    const long long p = off[(long long)digit * ntiles + blockIdx.x] + wc[warp][digit] + __popc(below);
    keys_out[p] = key;
    vals_out[p] = vals[i];
}

// common prefix length of sorted keys i and j, extended by the positions when the keys are equal; -1 outside [0, n)
__device__ __forceinline__ int delta(const unsigned* __restrict__ k, long long n, long long i, long long j) {
    if (j < 0 || j >= n) return -1;
    const unsigned a = k[i], b = k[j];
    return a == b ? 32 + __clz((unsigned)i ^ (unsigned)j) : __clz(a ^ b);
}

__global__ void __launch_bounds__(kThreads) k_rc_internal(int F, Ws W) {
    const long long i = thread_index();
    const long long n = F;
    if (i >= n - 1) return;
    const unsigned* k = W.keys0;
    const int d = delta(k, n, i, i + 1) - delta(k, n, i, i - 1) > 0 ? 1 : -1;
    const int dmin = delta(k, n, i, i - d);
    long long lmax = 2;
    while (delta(k, n, i, i + lmax * d) > dmin) lmax *= 2;
    long long l = 0;
    for (long long t = lmax / 2; t >= 1; t /= 2)
        if (delta(k, n, i, i + (l + t) * d) > dmin) l += t;
    const long long j = i + l * d;
    const int dnode = delta(k, n, i, j);
    long long s = 0, t = l;
    do {
        t = (t + 1) >> 1;
        if (delta(k, n, i, i + (s + t) * d) > dnode) s += t;
    } while (t > 1);
    const long long g = i + s * d + (d < 0 ? -1 : 0);
    const long long lo = i < j ? i : j, hi = i < j ? j : i;
    const int c0 = (int)(lo == g ? (n - 1) + g : g), c1 = (int)(hi == g + 1 ? (n - 1) + g + 1 : g + 1);
    W.nodes[i].d = make_int4(c0, c1, 0, 0);
    W.parent[c0] = (int)(i << 1);
    W.parent[c1] = (int)(i << 1) | 1;
}

__device__ __forceinline__ void put_box(Node* nd, int slot, float3 lo, float3 hi) {
    float* p = reinterpret_cast<float*>(nd) + 6 * slot;
    p[0] = lo.x; p[1] = lo.y; p[2] = lo.z; p[3] = hi.x; p[4] = hi.y; p[5] = hi.z;
}

__global__ void __launch_bounds__(kThreads) k_rc_leaves(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces, Ws W) {
    const long long i = thread_index();
    if (i >= F) return;
    const int3 t = load_face(faces, W.vals0[i]);
    float3 a, b, c;
    if (in_range(t, V)) {
        a = load3(verts, t.x);
        b = load3(verts, t.y);
        c = load3(verts, t.z);
    } else {                                                  // refused by the caller; never hit, empty box
        a = b = c = make_float3(__int_as_float(0x7fc00000), 0.0f, 0.0f);
    }
    W.tris[3 * i] = make_float4(a.x, a.y, a.z, b.x);
    W.tris[3 * i + 1] = make_float4(b.y, b.z, c.x, c.y);
    W.tris[3 * i + 2] = make_float4(c.z, 0.0f, 0.0f, 0.0f);
    float3 lo = make_float3(fminf(fminf(a.x, b.x), c.x), fminf(fminf(a.y, b.y), c.y), fminf(fminf(a.z, b.z), c.z));
    float3 hi = make_float3(fmaxf(fmaxf(a.x, b.x), c.x), fmaxf(fmaxf(a.y, b.y), c.y), fmaxf(fmaxf(a.z, b.z), c.z));
    if (!in_range(t, V)) {
        lo = make_float3(INFINITY, INFINITY, INFINITY);
        hi = make_float3(-INFINITY, -INFINITY, -INFINITY);
    }
    long long node = (F - 1) + i;
    while (node != 0) {                                       // the root is internal node 0 (a single leaf when F = 1)
        const int pp = W.parent[node];
        const int p = pp >> 1;
        put_box(W.nodes + p, pp & 1, lo, hi);
        __threadfence();
        if (atomicAdd(W.flags + p, 1) == 0) return;          // the other child is not done yet; it goes on
        const float* q = reinterpret_cast<const float*>(W.nodes + p);
        float x[12];
        for (int k = 0; k < 12; k++) x[k] = __ldcg(q + k);
        lo = make_float3(fminf(x[0], x[6]), fminf(x[1], x[7]), fminf(x[2], x[8]));
        hi = make_float3(fmaxf(x[3], x[9]), fmaxf(x[4], x[10]), fmaxf(x[5], x[11]));
        node = p;
    }
}

// ---------------------------------------------------------------- traversal
__device__ __forceinline__ float axis(float3 v, int k) { return k == 0 ? v.x : (k == 1 ? v.y : v.z); }

// the ray's parameter interval in the padded box meets [tnear, tfar]; conservative (see the header). t0: the entry, max(tnear, slab starts)
__device__ __forceinline__ bool box_hit(const float* b, float3 o, float3 d, float3 inv, float tnear, float tfar, float pad, float& t0) {
    t0 = tnear;
    float t1 = tfar;
    for (int k = 0; k < 3; k++) {
        const float lo = b[k] - pad, hi = b[3 + k] + pad, ok = axis(o, k), dk = axis(d, k), ik = axis(inv, k);
        if (dk == 0.0f) {
            if (!(ok >= lo && ok <= hi)) return false;
        } else if (fabsf(ik) <= 3.4e38f) {                    // a subnormal direction has no finite inverse: that axis is not used
            const float ta = (lo - ok) * ik, tb = (hi - ok) * ik;
            t0 = fmaxf(t0, fminf(ta, tb));
            t1 = fminf(t1, fmaxf(ta, tb));
        }
    }
    return t0 <= t1 + fabsf(t1) * kSlabRel;
}

__device__ __forceinline__ bool leaf_hit(const Ws& W, long long i, float3 o, float3 d, float tnear, float tfar) {
    float3 p0, p1, p2;
    leaf_corners(W, i, p0, p1, p2);
    float t, u, v;
    return hit_triangle(p0, p1, p2, o, d, tnear, tfar, t, u, v);
}

__device__ __forceinline__ float box_pad(float3 o, float scale) { return kPad * (scale + fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fabsf(o.z))); }

__device__ bool any_hit(const Ws& W, int F, float3 o, float3 d, float tnear, float tfar, float scale) {
    if (F == 0) return false;
    if (F == 1) return leaf_hit(W, 0, o, d, tnear, tfar);
    const float pad = box_pad(o, scale);
    const float3 inv = make_float3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    const int nl = F - 1;                                     // children at or above nl are leaves
    int stack[kStack];
    int sp = 0, node = 0;
    while (true) {
        const Node* nd = W.nodes + node;
        const float4 a = __ldg(&nd->a), b = __ldg(&nd->b), c = __ldg(&nd->c);
        const int4 ch = __ldg(&nd->d);
        const float b0[6] = {a.x, a.y, a.z, a.w, b.x, b.y}, b1[6] = {b.z, b.w, c.x, c.y, c.z, c.w};
        float e0, e1;
        bool h0 = box_hit(b0, o, d, inv, tnear, tfar, pad, e0), h1 = box_hit(b1, o, d, inv, tnear, tfar, pad, e1);
        if (h0 && ch.x >= nl) {
            if (leaf_hit(W, ch.x - nl, o, d, tnear, tfar)) return true;
            h0 = false;
        }
        if (h1 && ch.y >= nl) {
            if (leaf_hit(W, ch.y - nl, o, d, tnear, tfar)) return true;
            h1 = false;
        }
        if (h0 && h1) {
            stack[sp++] = ch.y;
            node = ch.x;
        } else if (h0 || h1) {
            node = h0 ? ch.x : ch.y;
        } else {
            if (sp == 0) return false;
            node = stack[--sp];
        }
    }
}

__global__ void __launch_bounds__(kThreads) k_rc_occluded(int F, long long R, const float* __restrict__ origins, const float* __restrict__ dirs,
                                                          float tnear, float tfar, Ws W, uint8_t* __restrict__ hit) {
    const long long r = thread_index();
    if (r >= R) return;
    hit[r] = any_hit(W, F, load3(origins, r), load3(dirs, r), tnear, tfar, mesh_scale(W)) ? 1 : 0;
}

// ---------------------------------------------------------------- first hits
struct Hit {
    float t;
    int face;                                                 // original index; -1: no hit
    float u, v;
};

// sorted leaf i under the caller's (tnear, tfar): taken when its t is smaller, or equal with a smaller original face
__device__ __forceinline__ void visit_first(const Ws& W, long long i, float3 o, float3 d, float tnear, float tfar, Hit& best) {
    float3 p0, p1, p2;
    leaf_corners(W, i, p0, p1, p2);
    float t, u, v;
    if (!hit_triangle(p0, p1, p2, o, d, tnear, tfar, t, u, v) || t > best.t) return;
    const int f = __ldg(W.vals0 + i);
    if (t == best.t && f > best.face) return;
    best = Hit{t, f, u, v};
}

// the smallest passing t, ties to the smallest face: that of testing every face. Nearer child first by the slab entry (child 0 on a tie);
// a box is skipped when the slab test fails against (tnear, min(tfar, best t)), which is non-strict, so boxes holding a tie are visited.
// A popped node is skipped when its stored entry fails that test's bound against the best t of now (x + |x| 2^-20 is monotone in x).
__device__ Hit first_hit(const Ws& W, int F, float3 o, float3 d, float tnear, float tfar, float scale) {
    Hit best{INFINITY, -1, 0.0f, 0.0f};
    if (F == 0) return best;
    if (F == 1) {
        visit_first(W, 0, o, d, tnear, tfar, best);
        return best;
    }
    const float pad = box_pad(o, scale);
    const float3 inv = make_float3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    const int nl = F - 1;
    int stack[kStack];
    float tstack[kStack];
    int sp = 0, node = 0;
    while (true) {
        const Node* nd = W.nodes + node;
        const float4 a = __ldg(&nd->a), b = __ldg(&nd->b), c = __ldg(&nd->c);
        const int4 ch = __ldg(&nd->d);
        const float b0[6] = {a.x, a.y, a.z, a.w, b.x, b.y}, b1[6] = {b.z, b.w, c.x, c.y, c.z, c.w};
        const float cap = fminf(tfar, best.t);
        float e0, e1;
        const bool g0 = box_hit(b0, o, d, inv, tnear, cap, pad, e0), g1 = box_hit(b1, o, d, inv, tnear, cap, pad, e1);
        const bool swap = g0 && g1 ? e1 < e0 : false;
        const int n0 = swap ? ch.y : ch.x, n1 = swap ? ch.x : ch.y;
        bool h0 = swap ? g1 : g0, h1 = swap ? g0 : g1;
        const float f1 = swap ? e0 : e1;
        if (h0 && n0 >= nl) {
            visit_first(W, n0 - nl, o, d, tnear, tfar, best);
            h0 = false;
        }
        if (h1 && n1 >= nl) {
            visit_first(W, n1 - nl, o, d, tnear, tfar, best);
            h1 = false;
        }
        if (h0 && h1) {
            stack[sp] = n1;
            tstack[sp++] = f1;
            node = n0;
        } else if (h0 || h1) {
            node = h0 ? n0 : n1;
        } else {
            float bound;
            do {
                if (sp == 0) return best;
                --sp;
                const float cp = fminf(tfar, best.t);
                bound = cp + fabsf(cp) * kSlabRel;
            } while (tstack[sp] > bound);
            node = stack[sp];
        }
    }
}

__global__ void __launch_bounds__(kThreads) k_fh_rays(int F, long long R, const float* __restrict__ origins, const float* __restrict__ dirs,
                                                           float tnear, float tfar, Ws W, float* __restrict__ t_out, int* __restrict__ face_out,
                                                           float* __restrict__ bary_out) {
    const long long r = thread_index();
    if (r >= R) return;
    const Hit h = first_hit(W, F, load3(origins, r), load3(dirs, r), tnear, tfar, mesh_scale(W));
    const bool hit = h.face >= 0;
    t_out[r] = h.t;
    face_out[r] = h.face;
    bary_out[3 * r] = hit ? (1.0f - h.u) - h.v : 0.0f;
    bary_out[3 * r + 1] = hit ? h.u : 0.0f;
    bary_out[3 * r + 2] = hit ? h.v : 0.0f;
}

// ---------------------------------------------------------------- rendering
#ifndef PSDF_RENDER_ROWS
constexpr bool kRenderTiles = true;
#else
constexpr bool kRenderTiles = false;                          // row order: built only by tools/bench_mesh_render.py, to measure against
#endif
constexpr int kTileW = 8, kTileH = 4;                         // the pixels of one warp

struct RenderOut {
    float* rgb;                                               // [I,3,H,W]
    float* mask;                                              // [I,1,H,W]
    float* depth;                                             // [I,1,H,W]
    float* normal;                                            // [I,3,H,W]
    int* face;                                                // [I,1,H,W]
};

__device__ __forceinline__ float3 blend(const float* __restrict__ a, int3 t, float b0, float b1, float b2) {
    const float3 x = load3(a, t.x), y = load3(a, t.y), z = load3(a, t.z);
    return make_float3((b0 * x.x + b1 * y.x) + b2 * z.x, (b0 * x.y + b1 * y.y) + b2 * z.y, (b0 * x.z + b1 * y.z) + b2 * z.z);
}

// thread g -> (image, x, y): a warp takes one 8 x 4 tile (tiles row by row, image by image), or in row order 32 consecutive pixels
// (at least 4 blocks per SM: without that minimum ptxas keeps it to 48 registers and spills; with it, 56 and no spills)
template <bool kTiles>
__global__ void __launch_bounds__(kThreads, 4) k_fh_render(int F, int I, int H, int Wd, const float* __restrict__ verts,
                                                        const int* __restrict__ faces, const float* __restrict__ normals,
                                                        const float* __restrict__ colors, const float* __restrict__ K,
                                                        const float* __restrict__ tf, float tnear, float tfar, Ws W, RenderOut out) {
    const long long g = thread_index();
    long long im;
    int x, y;
    if (kTiles) {
        const long long tx = (Wd + kTileW - 1) / kTileW, per = tx * ((H + kTileH - 1) / kTileH) * 32;
        im = g / per;
        const long long q = g - im * per, tile = q >> 5;
        const int lane = (int)(q & 31);
        x = (int)(tile % tx) * kTileW + (lane & (kTileW - 1));
        y = (int)(tile / tx) * kTileH + (lane >> 3);
        if (im >= I || x >= Wd || y >= H) return;
    } else {
        const long long plane = (long long)H * Wd;
        im = g / plane;
        if (im >= I) return;
        const int p = (int)(g - im * plane);
        x = p % Wd;
        y = p / Wd;
    }
    float3 o, d;
    reel_ray((float)x + 0.5f, (float)y + 0.5f, K + 9 * im, tf + 16 * im, o, d);
    const Hit h = first_hit(W, F, o, d, tnear, tfar, mesh_scale(W));
    float3 n = make_float3(0.0f, 0.0f, 0.0f), rgb = n;
    float depth = 0.0f;
    if (h.face >= 0) {
        const int3 t = load_face(faces, h.face);
        const float b0 = (1.0f - h.u) - h.v, b1 = h.u, b2 = h.v;
        if (normals) {
            n = blend(normals, t, b0, b1, b2);
        } else {
            const float3 a = load3(verts, t.x);
            n = cross3(sub3(load3(verts, t.y), a), sub3(load3(verts, t.z), a));
        }
        const float l = sqrtf(dot3(n, n));
        n = l == 0.0f ? make_float3(0.0f, 0.0f, 0.0f) : make_float3(n.x / l, n.y / l, n.z / l);
        rgb = colors ? blend(colors, t, b0, b1, b2) : make_float3(0.5f + 0.5f * n.x, 0.5f + 0.5f * n.y, 0.5f + 0.5f * n.z);
        depth = h.t;
    }
    const long long plane = (long long)H * Wd, p = (long long)y * Wd + x;
    if (out.rgb) {
        float* q = out.rgb + 3 * im * plane + p;
        q[0] = rgb.x; q[plane] = rgb.y; q[2 * plane] = rgb.z;
    }
    if (out.normal) {
        float* q = out.normal + 3 * im * plane + p;
        q[0] = n.x; q[plane] = n.y; q[2 * plane] = n.z;
    }
    if (out.mask) out.mask[im * plane + p] = h.face >= 0 ? 1.0f : 0.0f;
    if (out.depth) out.depth[im * plane + p] = depth;
    if (out.face) out.face[im * plane + p] = h.face;
}

__global__ void __launch_bounds__(kThreads) k_rc_ao(int V, int F, int S, const float* __restrict__ verts, const float* __restrict__ normals,
                                                    const float* __restrict__ dirs, Ws W) {
    const long long r = thread_index();
    if (r >= (long long)V * S) return;
    const long long i = r / S, s = r - i * S;
    float3 d = load3(dirs, s);
    if (dot3(d, load3(normals, i)) < 0.0f) d = make_float3(-d.x, -d.y, -d.z);
    if (any_hit(W, F, load3(verts, i), d, 1e-4f, INFINITY, mesh_scale(W))) atomicAdd(W.hits + i, 1);
}

__global__ void __launch_bounds__(kThreads) k_rc_vis(int V, int S, Ws W, float* __restrict__ vis) {
    const long long i = thread_index();
    if (i < V) vis[i] = (float)(S - W.hits[i]) / (float)S;
}
}  // namespace

extern "C" {

long long psdf_mesh_bvh_workspace_bytes(long long nr_vertices, long long nr_faces) {
    if (nr_vertices < 0 || nr_faces < 0) return PSDF_ERR_ARG;
    if (nr_vertices > kIntMax || nr_faces > kIntMax) return PSDF_ERR_UNSUPPORTED;
    return carve(nullptr, nr_vertices, nr_faces, nullptr);
}

int psdf_mesh_bvh_build(int V, int F, const float* verts, const int* faces, uint8_t* workspace, void* stream) {
    if (V < 0 || F < 0 || !workspace || (F > 0 && !faces) || (V > 0 && !verts)) return PSDF_ERR_ARG;
    Ws W;
    carve(workspace, V, F, &W);
    cudaMemsetAsync(W.info, 0, kHeaderBytes, ST);
    cudaMemsetAsync(W.bounds, 0xff, 12, ST);
    cudaMemsetAsync(W.bounds + 3, 0, 20, ST);
    if (F > 0) {
        k_mesh_check<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
        k_rc_bounds<<<blocks(F), kThreads, 0, ST>>>(V, F, verts, faces, W);
        k_rc_morton<<<blocks(F), kThreads, 0, ST>>>(V, F, verts, faces, W);
    }
    if (F > 1) {
        const long long nt = ntiles_of(F);
        unsigned* k[2] = {W.keys0, W.keys1};
        int* v[2] = {W.vals0, W.vals1};
        for (int pass = 0; pass < 4; pass++) {                // bits 0-7, 8-15, 16-23, 24-29; ends in keys0 / vals0
            const int a = pass & 1, shift = 8 * pass;
            k_rc_hist<<<(unsigned)nt, kThreads, 0, ST>>>(F, k[a], shift, W.hist, nt);
            scan<Count>(W.hist, kDigits * nt, W.tiles, W.off, ST);
            k_rc_scatter<<<(unsigned)nt, kThreads, 0, ST>>>(F, k[a], v[a], shift, W.off, nt, k[1 - a], v[1 - a]);
        }
        k_rc_internal<<<blocks(F - 1), kThreads, 0, ST>>>(F, W);
        cudaMemsetAsync(W.flags, 0, 4 * (size_t)(F - 1), ST);
    }
    if (F > 0) k_rc_leaves<<<blocks(F), kThreads, 0, ST>>>(V, F, verts, faces, W);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_occluded(int V, int F, long long R, const float* origins, const float* dirs, float tnear, float tfar,
                       const uint8_t* workspace, uint8_t* hit_out, void* stream) {
    if (V < 0 || F < 0 || R < 0 || !workspace || (R > 0 && (!origins || !dirs || !hit_out))) return PSDF_ERR_ARG;
    if (R > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    if (R == 0) return PSDF_OK;
    Ws W;
    carve(const_cast<uint8_t*>(workspace), V, F, &W);
    k_rc_occluded<<<blocks(R), kThreads, 0, ST>>>(F, R, origins, dirs, tnear, tfar, W, hit_out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_first_hit(int V, int F, long long R, const float* origins, const float* dirs, float tnear, float tfar, const uint8_t* workspace,
                        float* t_out, int* face_out, float* bary_out, void* stream) {
    if (V < 0 || F < 0 || R < 0 || !workspace || (R > 0 && (!origins || !dirs || !t_out || !face_out || !bary_out))) return PSDF_ERR_ARG;
    if (R > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    if (R == 0) return PSDF_OK;
    Ws W;
    carve(const_cast<uint8_t*>(workspace), V, F, &W);
    k_fh_rays<<<blocks(R), kThreads, 0, ST>>>(F, R, origins, dirs, tnear, tfar, W, t_out, face_out, bary_out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_render(int V, int F, const float* verts, const int* faces, const float* normals, const float* colors, int I, int H, int W_,
                     const float* K, const float* tf_world_cam, float tnear, float tfar, const uint8_t* workspace, float* rgb_out,
                     float* mask_out, float* depth_out, float* normal_out, int* face_out, void* stream) {
    if (V < 0 || F < 0 || I < 0 || H < 0 || W_ < 0 || !workspace) return PSDF_ERR_ARG;
    if ((F > 0 && (!verts || !faces)) || (I > 0 && (!K || !tf_world_cam))) return PSDF_ERR_ARG;
    const long long plane = (long long)H * W_;
    if (plane > kIntMax) return PSDF_ERR_UNSUPPORTED;
    const long long n = kRenderTiles ? (long long)I * psdf::div_up(W_, kTileW) * psdf::div_up(H, kTileH) * 32 : (long long)I * plane;
    if (n > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    if (I == 0 || plane == 0) return PSDF_OK;
    Ws W;
    carve(const_cast<uint8_t*>(workspace), V, F, &W);
    const RenderOut out{rgb_out, mask_out, depth_out, normal_out, face_out};
    k_fh_render<kRenderTiles><<<blocks(n), kThreads, 0, ST>>>(F, I, H, W_, verts, faces, normals, colors, K, tf_world_cam, tnear, tfar, W,
                                                               out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_ambient_occlusion(int V, int F, int S, const float* verts, const float* normals, const float* dirs, uint8_t* workspace,
                                float* vis_out, void* stream) {
    if (V < 0 || F < 0 || S < 1 || !workspace || (V > 0 && (!verts || !normals || !dirs || !vis_out))) return PSDF_ERR_ARG;
    if ((long long)V * S > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    if (V == 0) return PSDF_OK;
    Ws W;
    carve(workspace, V, F, &W);
    cudaMemsetAsync(W.hits, 0, 4 * (size_t)V, ST);
    k_rc_ao<<<blocks((long long)V * S), kThreads, 0, ST>>>(V, F, S, verts, normals, dirs, W);
    k_rc_vis<<<blocks(V), kThreads, 0, ST>>>(V, S, W, vis_out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
