// The linear BVH over the faces of an indexed triangle mesh, sm_90a: its workspace and its build. The ray, distance and winding queries
// (mesh_raycast.cu, mesh_distance.cu, mesh_winding.cu) read the tree through mesh_bvh.cuh. Built with -fmad=false, as its users are.
//
// Build (psdf_mesh_bvh_build): the centroids' bounds and the largest |coordinate| are reduced with ordered-key atomics (k_bvh_bounds);
// each face gets the 30-bit Morton code of its centroid within those bounds (k_bvh_morton); four stable 8-bit LSD radix passes
// (k_bvh_hist, the int64 scan of mesh_csr.cuh over the digit-major tile histogram, k_bvh_scatter) sort the faces by code; Karras' radix
// tree over the sorted codes, ties broken by sorted position, gives the F - 1 internal nodes (k_bvh_internal); k_bvh_leaves writes each
// leaf's triangle in sorted order and refits the boxes bottom-up, the second child to arrive at a node going on.
//
//   k_bvh_bounds     centroid bounds and max |coordinate| of the valid faces                          thread per face
//   k_bvh_morton     Morton code and face index                                                      thread per face
//   k_bvh_hist       per-tile counts of one 8-bit digit, digit-major                                 tile of 256 faces
//   k_bvh_scatter    stable scatter of one digit                                                     tile of 256 faces
//   k_bvh_internal   children and parents of internal node i (Karras 2012)                            thread per internal node
//   k_bvh_leaves     leaf triangles and the bottom-up box refit                                       thread per leaf
#include "mesh_bvh.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ unsigned float_key(float f) {
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__device__ __forceinline__ float3 centroid(float3 a, float3 b, float3 c) {
    const float k = 1.0f / 3.0f;
    return make_float3(((a.x + b.x) + c.x) * k, ((a.y + b.y) + c.y) * k, ((a.z + b.z) + c.z) * k);
}

__global__ void __launch_bounds__(kThreads) k_bvh_bounds(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces, Ws W) {
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

__global__ void __launch_bounds__(kThreads) k_bvh_morton(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces, Ws W) {
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

__global__ void __launch_bounds__(kThreads) k_bvh_hist(int F, const unsigned* __restrict__ keys, int shift, int* __restrict__ hist,
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
__global__ void __launch_bounds__(kThreads) k_bvh_scatter(int F, const unsigned* __restrict__ keys, const int* __restrict__ vals, int shift,
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

__global__ void __launch_bounds__(kThreads) k_bvh_internal(int F, Ws W) {
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

__global__ void __launch_bounds__(kThreads) k_bvh_leaves(int V, int F, const float* __restrict__ verts, const int* __restrict__ faces, Ws W) {
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
    // the node's box goes into its parent's slot before the arrival; the second child reads both slots back
    climb(W, F, i, W.flags, [&](int p, int slot) { put_box(W.nodes + p, slot, lo, hi); }, [&](int p) {
        const float* q = reinterpret_cast<const float*>(W.nodes + p);
        float x[12];
        for (int k = 0; k < 12; k++) x[k] = __ldcg(q + k);
        lo = make_float3(fminf(x[0], x[6]), fminf(x[1], x[7]), fminf(x[2], x[8]));
        hi = make_float3(fmaxf(x[3], x[9]), fmaxf(x[4], x[10]), fmaxf(x[5], x[11]));
    });
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
        k_bvh_bounds<<<blocks(F), kThreads, 0, ST>>>(V, F, verts, faces, W);
        k_bvh_morton<<<blocks(F), kThreads, 0, ST>>>(V, F, verts, faces, W);
    }
    if (F > 1) {
        const long long nt = ntiles_of(F);
        unsigned* k[2] = {W.keys0, W.keys1};
        int* v[2] = {W.vals0, W.vals1};
        for (int pass = 0; pass < 4; pass++) {                // bits 0-7, 8-15, 16-23, 24-29; ends in keys0 / vals0
            const int a = pass & 1, shift = 8 * pass;
            k_bvh_hist<<<(unsigned)nt, kThreads, 0, ST>>>(F, k[a], shift, W.hist, nt);
            scan<Count>(W.hist, kDigits * nt, W.tiles, W.off, ST);
            k_bvh_scatter<<<(unsigned)nt, kThreads, 0, ST>>>(F, k[a], v[a], shift, W.off, nt, k[1 - a], v[1 - a]);
        }
        k_bvh_internal<<<blocks(F - 1), kThreads, 0, ST>>>(F, W);
        cudaMemsetAsync(W.flags, 0, 4 * (size_t)(F - 1), ST);
    }
    if (F > 0) k_bvh_leaves<<<blocks(F), kThreads, 0, ST>>>(V, F, verts, faces, W);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
