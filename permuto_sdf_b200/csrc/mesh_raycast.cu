// Any-hit and first-hit ray casting against an indexed triangle mesh through the BVH of mesh_bvh.cu, per-vertex ambient occlusion and
// rendering from reel cameras, sm_90a. Built with -fmad=false: the ray-triangle test is rounded operation by operation as
// include/psdf_b200.h states it, so oracle/raycast.py and, for first hits, tests/first_hit_oracle.py (brute force over all triangles)
// reproduce every answer. The tree only decides which triangles are tested; the answer is "some triangle passes", or for first hits the
// passing triangle of smallest t, ties to the smallest original face index. Both queries walk the tree with traverse (mesh_bvh.cuh).
//
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

// ---------------------------------------------------------------- traversal
__device__ __forceinline__ float axis(float3 v, int k) { return k == 0 ? v.x : (k == 1 ? v.y : v.z); }

// the ray's parameter interval in the padded box meets [tnear, tfar]; conservative (see the header). t0: the entry, max(tnear, slab starts)
__device__ __forceinline__ bool box_hit(const Box& b, float3 o, float3 d, float3 inv, float tnear, float tfar, float pad, float& t0) {
    t0 = tnear;
    float t1 = tfar;
    for (int k = 0; k < 3; k++) {
        const float lo = axis(b.lo, k) - pad, hi = axis(b.hi, k) + pad, ok = axis(o, k), dk = axis(d, k), ik = axis(inv, k);
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

__device__ __forceinline__ float box_pad(float3 o, float scale) { return kPad * (scale + fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fabsf(o.z))); }

// what both ray queries hold for the walk: the ray, its reciprocal direction and its box padding
struct Ray {
    const Ws& W;
    float3 o, d, inv;
    float tnear, tfar, pad;
    __device__ Ray(const Ws& W, float3 o, float3 d, float tnear, float tfar, float scale)
        : W(W), o(o), d(d), inv(make_float3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z)), tnear(tnear), tfar(tfar), pad(box_pad(o, scale)) {}
};

// any hit (traverse): no order, every key 0, so child 0 goes first; no bound to tighten; the first passing leaf ends the walk
struct AnyHit : Ray {
    using Ray::Ray;
    bool hit = false;
    __device__ bool enter(const Box& b, float& key) const {
        float t0;
        key = 0.0f;
        return box_hit(b, o, d, inv, tnear, tfar, pad, t0);
    }
    __device__ bool visit(long long i) {
        float3 p0, p1, p2;
        leaf_corners(W, i, p0, p1, p2);
        float t, u, v;
        hit = hit_triangle(p0, p1, p2, o, d, tnear, tfar, t, u, v);
        return hit;
    }
    __device__ bool keep(float) const { return true; }
};

__device__ bool any_hit(const Ws& W, int F, float3 o, float3 d, float tnear, float tfar, float scale) {
    AnyHit q(W, o, d, tnear, tfar, scale);
    traverse(W, F, q);
    return q.hit;
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

// first hit (traverse): the smallest passing t, ties to the smallest face, as testing every face gives. The key is the slab entry; a box
// enters when the slab test passes against (tnear, min(tfar, best t)), which is non-strict, so boxes holding a tie are visited. keep is
// that test's last comparison against the best t of now (x + |x| 2^-20 is monotone in x, and the entry does not depend on the cap), so
// it drops only boxes the test would now refuse. Leaves use the caller's (tnear, tfar).
struct FirstHit : Ray {
    using Ray::Ray;
    Hit best{INFINITY, -1, 0.0f, 0.0f};
    __device__ float cap() const { return fminf(tfar, best.t); }
    __device__ bool enter(const Box& b, float& key) const { return box_hit(b, o, d, inv, tnear, cap(), pad, key); }
    // sorted leaf i: taken when its t is smaller, or equal with a smaller original face
    __device__ bool visit(long long i) {
        float3 p0, p1, p2;
        leaf_corners(W, i, p0, p1, p2);
        float t, u, v;
        if (!hit_triangle(p0, p1, p2, o, d, tnear, tfar, t, u, v) || t > best.t) return false;
        const int f = __ldg(W.vals0 + i);
        if (t == best.t && f > best.face) return false;
        best = Hit{t, f, u, v};
        return false;
    }
    __device__ bool keep(float key) const {
        const float c = cap();
        return !(key > c + fabsf(c) * kSlabRel);
    }
};

__device__ Hit first_hit(const Ws& W, int F, float3 o, float3 d, float tnear, float tfar, float scale) {
    FirstHit q(W, o, d, tnear, tfar, scale);
    traverse(W, F, q);
    return q.best;
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
