// Midpoint and Loop subdivision of an indexed triangle mesh, sm_90a. Built with -fmad=false: every fp32 operation is rounded as written,
// so oracle/subdivide.py reproduces the output bit for bit. The rules (edges, their numbering, faces, positions) are stated in
// include/psdf_b200.h; this file only adds how they are computed.
//
// Vertex -> face CSR (mesh_csr.cuh): k_mesh_degree counts the faces of each vertex, the scan k_mesh_scan_* turns the counts into int64
// offsets, and k_sd_fill places each face in its vertices' lists with atomics, together with the two other corners of the face (the
// vertex's neighbours in it) at twice the offset. The face lists stay as filled (every use of them is order-free); k_sd_sort sorts each
// vertex's neighbour list, so that the Loop rule sums the neighbours in ascending index and a neighbour appears there once per face of the
// edge between them. The edge numbering is an exclusive scan of the corners that own their edge, with the same kernels. Faces with an
// index outside [0, V) or a repeated vertex are counted by k_mesh_check and never enter the CSR.
//
//   k_sd_fill      adj[off[v] + cursor] = f, nb[2 (off[v] + cursor) ..] = the other two corners   thread per face
//   k_sd_edge      own[c] = the smallest corner id of c's edge                                    thread per corner
//   k_sd_sort      heap sort of each vertex's neighbour list (Loop only)                          thread per vertex
//   k_sd_even      the old vertices: copied (midpoint) or moved by the Loop even rule              thread per vertex
//   k_sd_odd       the edge vertex of every owning corner                                          thread per corner
//   k_sd_faces     the four faces of every face                                                    thread per face
#include "mesh_csr.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
// workspace sections in order
struct Ws {
    long long* info;          // {faces outside [0, V), faces repeating a vertex, edges, 0}
    long long* off;           // [V + 1] CSR offsets
    int* deg;                 // [V] face count, then the fill cursor
    int* adj;                 // [3F] faces of each vertex
    int* nb;                  // [6F] the other two corners of each of those faces
    long long* tiles;         // [tiles + 1] tile sums of the scans
    int* own;                 // [3F] smallest corner id of each corner's edge (-1 for a corner of a bad face)
    long long* pos;           // [3F + 1] exclusive prefix of the owning corners: edge ids
};

long long carve(void* ws, long long V, long long F, Ws* W) {
    Sections s{static_cast<char*>(ws)};
    Ws w;
    s.take(w.info, kHeaderBytes);
    s.take(w.off, 8 * (V + 1));
    s.take(w.deg, 4 * V);
    s.take(w.adj, 12 * F);
    s.take(w.nb, 24 * F);
    s.take(w.tiles, 8 * tile_sums(V + 1 > 3 * F ? V + 1 : 3 * F));
    s.take(w.own, 12 * F);
    s.take(w.pos, 8 * (3 * F + 1));
    if (W) *W = w;
    return s.size;
}

__device__ __forceinline__ void store3(float* __restrict__ verts, long long v, float3 p) {
    verts[3 * v] = p.x;
    verts[3 * v + 1] = p.y;
    verts[3 * v + 2] = p.z;
}

// ---------------------------------------------------------------- the CSR and the edges
// the scanned value of the edge numbering: 1 for a corner that owns its edge
struct Owns {
    __device__ __forceinline__ long long operator()(int own, long long i) const { return own == i; }
};

__global__ void __launch_bounds__(kThreads) k_sd_fill(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    if (f >= F) return;
    const int3 t = load_face(faces, f);
    if (!valid(t, V)) return;
    for (int k = 0; k < 3; k++) {
        const int v = corner(t, k);
        const long long i = W.off[v] + atomicAdd(W.deg + v, 1);
        W.adj[i] = (int)f;
        W.nb[2 * i] = corner(t, k == 2 ? 0 : k + 1);
        W.nb[2 * i + 1] = corner(t, k == 0 ? 2 : k - 1);
    }
}

// the faces that hold the undirected edge {u, v} (both orders; a valid face holds it at one corner at most): their number, the smallest
// of those corner ids, and the opposite vertex of the last such face other than f. The list of the end with fewer faces is scanned.
struct Edge { int count; int min_corner; int other; };
__device__ Edge find_edge(const Ws& W, const int* __restrict__ faces, int u, int v, long long f) {
    Edge r{0, 0x7fffffff, -1};
    const int s = nr_faces(W, v) < nr_faces(W, u) ? v : u;
    for (long long i = W.off[s], e = W.off[s + 1]; i < e; i++) {
        const int h = W.adj[i];
        const int3 t = load_face(faces, h);
        for (int q = 0; q < 3; q++) {
            const int a = corner(t, q), b = corner(t, q == 2 ? 0 : q + 1);
            if ((a == u && b == v) || (a == v && b == u)) {
                r.count++;
                r.min_corner = min(r.min_corner, 3 * h + q);        // 3F < 2^31: checked by the entry points
                if (h != f) r.other = corner(t, q == 0 ? 2 : q - 1);
            }
        }
    }
    return r;
}

__global__ void __launch_bounds__(kThreads) k_sd_edge(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long c = thread_index();
    if (c >= 3LL * F) return;
    const long long f = c / 3;
    const int k = (int)(c - 3 * f);
    const int3 t = load_face(faces, f);
    if (!valid(t, V)) { W.own[c] = -1; return; }
    W.own[c] = find_edge(W, faces, corner(t, k), corner(t, k == 2 ? 0 : k + 1), f).min_corner;
}

__global__ void __launch_bounds__(kThreads) k_sd_sort(int V, Ws W) {
    const long long v = thread_index();
    if (v >= V) return;
    heap_sort(W.nb + 2 * W.off[v], 2 * (W.off[v + 1] - W.off[v]));
}

// ---------------------------------------------------------------- the new vertices and faces
__device__ __forceinline__ float3 add3(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 mul3(float s, float3 a) { return make_float3(s * a.x, s * a.y, s * a.z); }

// the Loop even rule over v's sorted neighbour list, in which each neighbour appears once per face of the edge
__device__ float3 loop_even(const Ws& W, const float* __restrict__ verts, int v) {
    const float3 p = load3(verts, v);
    const long long b = 2 * W.off[v], e = 2 * W.off[v + 1];
    if (b == e) return p;
    float3 s = make_float3(0.f, 0.f, 0.f);
    long long n = 0;
    int creases = 0, ca = -1, cb = -1;
    for (long long i = b; i < e;) {
        const int w = W.nb[i];
        long long j = i + 1;
        while (j < e && W.nb[j] == w) j++;
        n++;
        s = add3(s, load3(verts, w));
        if (j - i != 2) {
            creases++;
            if (creases == 1) ca = w; else cb = w;
        }
        i = j;
    }
    if (creases == 0) {
        const float beta = n == 3 ? 0.1875f : 3.0f / (float)(8 * n);
        const float wv = 1.0f - (float)n * beta;
        return add3(mul3(wv, p), mul3(beta, s));
    }
    if (creases == 2) return add3(mul3(0.75f, p), mul3(0.125f, add3(load3(verts, ca), load3(verts, cb))));
    return p;
}

__global__ void __launch_bounds__(kThreads) k_sd_even(int V, int smooth, const float* __restrict__ verts, Ws W, float* __restrict__ out) {
    const long long v = thread_index();
    if (v >= V) return;
    store3(out, v, smooth ? loop_even(W, verts, (int)v) : load3(verts, v));
}

__global__ void __launch_bounds__(kThreads) k_sd_odd(int V, int F, int smooth, const int* __restrict__ faces, const float* __restrict__ verts,
                                                     Ws W, float* __restrict__ out) {
    const long long c = thread_index();
    if (c >= 3LL * F || W.own[c] != c) return;
    const long long f = c / 3;
    const int k = (int)(c - 3 * f);
    const int3 t = load_face(faces, f);
    const int u = corner(t, k), v = corner(t, k == 2 ? 0 : k + 1);
    const float3 puv = add3(load3(verts, u), load3(verts, v));
    float3 p = mul3(0.5f, puv);
    if (smooth) {
        const Edge e = find_edge(W, faces, u, v, f);
        if (e.count == 2) {
            const int w = corner(t, k == 0 ? 2 : k - 1);
            p = add3(mul3(0.375f, puv), mul3(0.125f, add3(load3(verts, w), load3(verts, e.other))));
        }
    }
    store3(out, (long long)V + W.pos[c], p);
}

__global__ void __launch_bounds__(kThreads) k_sd_faces(int V, int F, const int* __restrict__ faces, Ws W, int* __restrict__ out) {
    const long long f = thread_index();
    if (f >= F) return;
    const int3 t = load_face(faces, f);
    if (!valid(t, V)) return;                                        // refused by the caller; its rows are left as they are
    const int e01 = (int)(V + W.pos[W.own[3 * f]]), e12 = (int)(V + W.pos[W.own[3 * f + 1]]), e20 = (int)(V + W.pos[W.own[3 * f + 2]]);
    int* o = out + 12 * f;
    o[0] = t.x; o[1] = e01; o[2] = e20;
    o[3] = e01; o[4] = t.y; o[5] = e12;
    o[6] = e20; o[7] = e12; o[8] = t.z;
    o[9] = e01; o[10] = e12; o[11] = e20;
}
}  // namespace

extern "C" {

long long psdf_mesh_subdivide_workspace_bytes(long long nr_vertices, long long nr_faces) {
    if (nr_vertices < 0 || nr_faces < 0) return PSDF_ERR_ARG;
    if (nr_vertices > kIntMax || 4 * nr_faces > kIntMax) return PSDF_ERR_UNSUPPORTED;
    return carve(nullptr, nr_vertices, nr_faces, nullptr);
}

int psdf_mesh_subdivide_count(int V, int F, const int* faces, uint8_t* workspace, void* stream) {
    if (V < 0 || F < 0 || 4LL * F > kIntMax || !workspace || (F > 0 && !faces)) return PSDF_ERR_ARG;
    Ws W;
    carve(workspace, V, F, &W);
    cudaMemsetAsync(W.info, 0, kHeaderBytes, ST);
    cudaMemsetAsync(W.deg, 0, 4 * (size_t)V, ST);
    if (F > 0) {
        k_mesh_check<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
        k_mesh_degree<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
    }
    scan<Count>(W.deg, V, W.tiles, W.off, ST);
    cudaMemsetAsync(W.deg, 0, 4 * (size_t)V, ST);
    if (F > 0) {
        k_sd_fill<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
        k_sd_edge<<<blocks(3LL * F), kThreads, 0, ST>>>(V, F, faces, W);
    }
    scan<Owns>(W.own, 3LL * F, W.tiles, W.pos, ST);
    cudaMemcpyAsync(W.info + 2, W.pos + 3LL * F, sizeof(long long), cudaMemcpyDeviceToDevice, ST);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_subdivide_emit(int V, int F, int smooth, const float* verts, const int* faces, uint8_t* workspace, float* verts_out,
                             int* faces_out, void* stream) {
    if (V < 0 || F < 0 || 4LL * F > kIntMax || !workspace || (V > 0 && (!verts || !verts_out)) || (F > 0 && (!faces || !faces_out)))
        return PSDF_ERR_ARG;
    Ws W;
    carve(workspace, V, F, &W);
    if (smooth && V > 0) k_sd_sort<<<blocks(V), kThreads, 0, ST>>>(V, W);
    if (V > 0) k_sd_even<<<blocks(V), kThreads, 0, ST>>>(V, smooth, verts, W, verts_out);
    if (F > 0) {
        k_sd_odd<<<blocks(3LL * F), kThreads, 0, ST>>>(V, F, smooth, faces, verts, W, verts_out);
        k_sd_faces<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W, faces_out);
    }
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
