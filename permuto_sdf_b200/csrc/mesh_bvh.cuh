// The linear BVH over the faces of an indexed triangle mesh, shared by mesh_raycast.cu (which builds it and casts rays) and
// mesh_distance.cu (closest points). The workspace layout, the node format and the box padding are stated in include/psdf_b200.h.
#pragma once
#include "mesh_csr.cuh"

namespace {
constexpr int kDigits = 256;                    // radix of the build's sort passes
constexpr int kStack = 64;                      // >= the internal nodes on any root-to-leaf path (<= 62, see the header)
constexpr float kPad = 1.0f / 4096.0f;         // box padding per unit of coordinate scale (see the header)

struct Node {                                   // internal node: the boxes of both children, then the children
    float4 a;                                   // lo0.xyz, hi0.x
    float4 b;                                   // hi0.yz, lo1.xy
    float4 c;                                   // lo1.z, hi1.xyz
    int4 d;                                     // child0, child1 (>= F - 1: leaf child - (F - 1)), 0, 0
};

struct Ws {
    long long* info;          // {faces outside [0, V), faces repeating a vertex, 0, 0}
    unsigned* bounds;         // ordered keys: centroid lo xyz, centroid hi xyz, max |coordinate|, 0
    unsigned* keys0;          // [F] Morton codes, sorted in place over the passes
    unsigned* keys1;          // [F]
    int* vals0;               // [F] face indices; after the build, the original face of each sorted leaf
    int* vals1;               // [F]
    int* hist;                // [256 ntiles] digit-major tile counts
    long long* off;           // [256 ntiles + 1] their exclusive prefix
    long long* tiles;         // scan tile sums
    Node* nodes;              // [F - 1]
    int* parent;              // [2F - 1] (parent << 1 | slot) of internal nodes, then of leaves
    int* flags;               // [F - 1] refit arrivals
    float4* tris;             // [3F] p0.xyz p1.x | p1.yz p2.xy | p2.z 0, in sorted order
    int* hits;                // [V] ambient occlusion hit counts
};

long long ntiles_of(long long F) { return (F + kThreads - 1) / kThreads; }

long long carve(void* ws, long long V, long long F, Ws* W) {
    Sections s{static_cast<char*>(ws)};
    Ws w;
    const long long nh = kDigits * ntiles_of(F);
    s.take(w.info, kHeaderBytes);
    s.take(w.bounds, 32);
    s.take(w.keys0, 4 * F);
    s.take(w.keys1, 4 * F);
    s.take(w.vals0, 4 * F);
    s.take(w.vals1, 4 * F);
    s.take(w.hist, 4 * nh);
    s.take(w.off, 8 * (nh + 1));
    s.take(w.tiles, 8 * tile_sums(nh));
    s.take(w.nodes, (long long)sizeof(Node) * (F > 1 ? F - 1 : 0));
    s.take(w.parent, 4 * (F > 0 ? 2 * F - 1 : 0));
    s.take(w.flags, 4 * (F > 1 ? F - 1 : 0));
    s.take(w.tris, 48 * F);
    s.take(w.hits, 4 * V);
    if (W) *W = w;
    return s.size;
}

// ---------------------------------------------------------------- fp32 arithmetic, rounded as written
__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
    return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// the largest |coordinate| of the mesh, which sets the box padding
__device__ __forceinline__ float mesh_scale(const Ws& W) { return __uint_as_float(W.bounds[6]); }

// the corners of sorted leaf i
__device__ __forceinline__ void leaf_corners(const Ws& W, long long i, float3& p0, float3& p1, float3& p2) {
    const float4 x = __ldg(W.tris + 3 * i), y = __ldg(W.tris + 3 * i + 1), z = __ldg(W.tris + 3 * i + 2);
    p0 = make_float3(x.x, x.y, x.z);
    p1 = make_float3(x.w, y.x, y.y);
    p2 = make_float3(y.z, y.w, z.x);
}
}  // namespace
