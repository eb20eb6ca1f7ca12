// The linear BVH over the faces of an indexed triangle mesh: its workspace, its node format, and the two walks over it. mesh_bvh.cu
// builds the tree; mesh_raycast.cu (any and first hits), mesh_distance.cu (closest points) and mesh_winding.cu (winding numbers) read it.
// traverse is the top-down walk of the ray and distance queries, climb the bottom-up one of the box refit and the winding moments. The
// workspace layout, the node format, the box padding and the traversal rules are stated in include/psdf_b200.h.
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

// ---------------------------------------------------------------- nodes
struct Box {
    float3 lo, hi;
};

// internal node i as a walk reads it: the boxes of both children and the children (>= F - 1: leaf child - (F - 1))
struct NodeView {
    Box box[2];
    int child[2];
};

__device__ __forceinline__ NodeView load_node(const Ws& W, int i) {
    const Node* nd = W.nodes + i;
    const float4 a = __ldg(&nd->a), b = __ldg(&nd->b), c = __ldg(&nd->c);
    const int4 d = __ldg(&nd->d);
    return NodeView{{{make_float3(a.x, a.y, a.z), make_float3(a.w, b.x, b.y)}, {make_float3(b.z, b.w, c.x), make_float3(c.y, c.z, c.w)}},
                    {d.x, d.y}};
}

// ---------------------------------------------------------------- top-down: one query, depth first
// The walk of query q over the tree, the same rule for every query. q supplies
//   enter(box, key)  whether to go into a child's box, and that child's order key;
//   visit(i)         visits sorted leaf i; true ends the walk;
//   keep(key)        whether a child entered with this key still passes the query's bound as it stands now.
// At a node both children's boxes are tested; the one of smaller key goes first only when both enter (child 0 on a tie). A first child
// that is a leaf is visited at once, and the second is then tested with keep again, since the visit may have tightened the bound. Of
// two internal children the second is pushed with its key; a popped node is skipped while !keep(key). Only internal nodes are pushed,
// at most one per level, so kStack entries hold any path (see the header).
template <class Q> __device__ __forceinline__ void traverse(const Ws& W, int F, Q& q) {
    if (F == 0) return;
    if (F == 1) {                                             // the root is leaf 0
        q.visit(0);
        return;
    }
    const int nl = F - 1;                                     // children at or above nl are leaves
    int stack[kStack];
    float kstack[kStack];
    int sp = 0, node = 0;
    while (true) {
        const NodeView nd = load_node(W, node);
        float k0, k1;
        const bool g0 = q.enter(nd.box[0], k0), g1 = q.enter(nd.box[1], k1);
        const bool swap = g0 && g1 && k1 < k0;
        const int n0 = swap ? nd.child[1] : nd.child[0], n1 = swap ? nd.child[0] : nd.child[1];
        bool h0 = swap ? g1 : g0, h1 = swap ? g0 : g1;
        const float f1 = swap ? k0 : k1;
        if (h0 && n0 >= nl) {
            if (q.visit(n0 - nl)) return;
            h0 = false;
            h1 = h1 && q.keep(f1);
        }
        if (h1 && n1 >= nl) {
            if (q.visit(n1 - nl)) return;
            h1 = false;
        }
        if (h0 && h1) {
            stack[sp] = n1;
            kstack[sp++] = f1;
            node = n0;
        } else if (h0 || h1) {
            node = h0 ? n0 : n1;
        } else {
            do {
                if (sp == 0) return;
                --sp;
            } while (!q.keep(kstack[sp]));
            node = stack[sp];
        }
    }
}

// ---------------------------------------------------------------- bottom-up: one thread per leaf
// The climb from sorted leaf i to the root, every internal node combined once, after both its children. At each parent p the child
// first calls publish(p, slot), with slot its side of p, and fences what it and the nodes below it wrote; then it arrives on flags[p].
// The first to arrive returns; the second calls combine(p), which reads both children's results with __ldcg (another thread of the
// same launch may have written them), and goes on from p. flags [F - 1] must be zero before the launch.
template <class Publish, class Combine>
__device__ __forceinline__ void climb(const Ws& W, int F, long long i, int* flags, Publish publish, Combine combine) {
    long long node = (F - 1) + i;
    while (node != 0) {                                       // the root is internal node 0 (a single leaf when F = 1)
        const int pp = W.parent[node];
        const int p = pp >> 1;
        publish(p, pp & 1);
        __threadfence();
        if (atomicAdd(flags + p, 1) == 0) return;            // the other child is not done yet; it goes on
        combine(p);
        node = p;
    }
}
}  // namespace
