// Connected components of the vertex graph of an indexed triangle mesh, sm_90a. Each face joins its three vertices.
//
// Lock-free union-find (in the style of ECL-CC): parent[v] = v to start; one pass over the faces finds the roots of a face's vertices with
// path halving and links the larger root under the smaller one with atomicCAS, retrying until they share a root; one pass of full
// compression then gives label[v] = root(v). A root is only ever linked under a smaller index and path halving only moves a vertex to an
// ancestor, so parent[v] <= v throughout and the final root of a component is its smallest vertex index. The labels are therefore a fixed
// function of the partition and the vertex numbering: the same bits for any face order, launch configuration and run, with no
// canonicalisation pass. Face counts, the component count and the largest component come from integer atomics, which are exact.
//
//   k_cc_init      parent[v] = v, face_counts[v] = 0, info = 0                                       thread per vertex
//   k_cc_link      validate a face's indices, unite its vertices                                      thread per face
//   k_cc_compress  label[v] = root(v), in place                                                       thread per vertex
//   k_cc_count     face_counts[label[f.x]] += 1 (warp-aggregated over equal labels)                   thread per face
//   k_cc_roots     components += 1 and largest = max((count << 32) | ~label) at every root            thread per vertex
//   k_cc_keep      keep[v] = face_counts[label[v]] >= min_faces, or label[v] == the largest's label   thread per vertex
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kThreads = 256;
constexpr long long kHeaderBytes = 256;          // info[4] (int64), padded so that the labels start 256-byte aligned
constexpr long long kIntMax = 0x7fffffffLL;
#define ST ((cudaStream_t)stream)

struct Ws {
    long long* info;                             // {components, faces with an index outside [0, V), largest key, unused}
    int* label;                                  // [V]: parent during linking, the label after compression
    int* count;                                  // [V]: faces per component, indexed by label
};

Ws carve(void* ws, int V) {
    char* p = static_cast<char*>(ws);
    Ws W;
    W.info = reinterpret_cast<long long*>(p);
    W.label = reinterpret_cast<int*>(p + kHeaderBytes);
    W.count = W.label + V;
    return W;
}

__device__ __forceinline__ long long thread_index() { return (long long)blockIdx.x * kThreads + threadIdx.x; }

// root of x with path halving: every vertex on the way is moved to its grandparent. Only non-roots are written (a root changes only by
// the CAS in unite), and every value stored is an ancestor, so concurrent halving and linking keep each vertex in its component. Loads
// go to L2 (ld.cg): a root linked by another SM is seen at the next load.
__device__ __forceinline__ int find_root(int* parent, int x) {
    int p = __ldcg(parent + x);
    while (p != x) {
        const int gp = __ldcg(parent + p);
        if (gp == p) return p;
        __stcg(parent + x, gp);
        x = gp;
        p = __ldcg(parent + x);
    }
    return x;
}

__device__ __forceinline__ void unite(int* parent, int a, int b) {
    int ra = find_root(parent, a), rb = find_root(parent, b);
    while (ra != rb) {
        const int hi = max(ra, rb), lo = min(ra, rb);
        const int old = atomicCAS(parent + hi, hi, lo);
        if (old == hi) return;
        // hi was linked under `old` in the meantime: continue from the two current roots
        ra = find_root(parent, old);
        rb = find_root(parent, lo);
    }
}

__device__ __forceinline__ bool face_ok(int3 f, int V) {
    return (unsigned)f.x < (unsigned)V && (unsigned)f.y < (unsigned)V && (unsigned)f.z < (unsigned)V;
}

__device__ __forceinline__ int3 load_face(const int* __restrict__ faces, long long i) {
    const int* p = faces + 3 * i;
    return make_int3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
}

__global__ void __launch_bounds__(kThreads) k_cc_init(int V, Ws W) {
    const long long v = thread_index();
    if (v < V) {
        W.label[v] = (int)v;
        W.count[v] = 0;
    }
    if (v < 4) W.info[v] = 0;
}

// faces with an index outside [0, V) are not linked (nothing out of range is read or written) and are counted in info[1]
__global__ void __launch_bounds__(kThreads) k_cc_link(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long i = thread_index();
    bool bad = false;
    if (i < F) {
        const int3 f = load_face(faces, i);
        if (face_ok(f, V)) {
            // the third edge (z, x) joins nothing the first two have not joined
            unite(W.label, f.x, f.y);
            unite(W.label, f.y, f.z);
        } else {
            bad = true;
        }
    }
    const unsigned m = __ballot_sync(kFullMask, bad);
    if (m && (threadIdx.x & 31) == 0) atomicAdd(reinterpret_cast<unsigned long long*>(W.info + 1), (unsigned long long)__popc(m));
}

// no link happens any more: every parent read is an ancestor (the old parent or the root another thread stored), roots do not change
__global__ void __launch_bounds__(kThreads) k_cc_compress(int V, Ws W) {
    const long long v = thread_index();
    if (v >= V) return;
    int r = __ldcg(W.label + v);
    for (int p = __ldcg(W.label + r); p != r; p = __ldcg(W.label + r)) r = p;
    W.label[v] = r;
}

// faces of a warp are mostly in one component: one atomic per distinct label in the warp
__global__ void __launch_bounds__(kThreads) k_cc_count(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long i = thread_index();
    int lab = -1;
    if (i < F) {
        const int3 f = load_face(faces, i);
        if (face_ok(f, V)) lab = __ldg(W.label + f.x);
    }
    const unsigned peers = __match_any_sync(kFullMask, lab);
    if (lab >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(W.count + lab, __popc(peers));
}

// the largest component: most faces, then the smallest label (the larger complement). V < 2^31 keeps ~label above 2^31 - 1, so a
// vertex set with no faces still has a non-zero key.
__global__ void __launch_bounds__(kThreads) k_cc_roots(int V, Ws W) {
    const long long v = thread_index();
    const bool root = v < V && __ldg(W.label + v) == (int)v;
    unsigned long long key = root ? ((unsigned long long)(unsigned)__ldg(W.count + v) << 32) | (unsigned)~(unsigned)v : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long k = __shfl_xor_sync(kFullMask, key, o);
        key = k > key ? k : key;
    }
    const unsigned m = __ballot_sync(kFullMask, root);
    if (m && (threadIdx.x & 31) == 0) {
        atomicAdd(reinterpret_cast<unsigned long long*>(W.info), (unsigned long long)__popc(m));
        atomicMax(reinterpret_cast<unsigned long long*>(W.info + 2), key);
    }
}

__global__ void __launch_bounds__(kThreads) k_cc_keep(int V, int largest, long long min_faces, Ws W, uint8_t* __restrict__ keep) {
    const long long v = thread_index();
    if (v >= V) return;
    const int lab = __ldg(W.label + v);
    bool k;
    if (largest) k = lab == (int)~(unsigned)__ldg(W.info + 2);          // the low word of the key is ~label
    else k = (long long)__ldg(W.count + lab) >= min_faces;
    keep[v] = (uint8_t)k;
}

unsigned blocks(long long n) { return (unsigned)(n > 0 ? div_up(n, kThreads) : 1); }
}  // namespace

extern "C" {

long long psdf_mesh_components_workspace_bytes(long long nr_vertices, long long nr_faces) {
    if (nr_vertices < 0 || nr_faces < 0) return PSDF_ERR_ARG;
    if (nr_vertices > kIntMax || nr_faces > kIntMax) return PSDF_ERR_UNSUPPORTED;
    return kHeaderBytes + 8LL * nr_vertices;
}

int psdf_mesh_components(int V, int F, const int* faces, uint8_t* workspace, void* stream) {
    if (V < 0 || F < 0 || !workspace || (F > 0 && !faces)) return PSDF_ERR_ARG;
    const Ws W = carve(workspace, V);
    k_cc_init<<<blocks(V), kThreads, 0, ST>>>(V, W);
    if (F > 0) k_cc_link<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
    if (V > 0) k_cc_compress<<<blocks(V), kThreads, 0, ST>>>(V, W);
    if (F > 0) k_cc_count<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
    if (V > 0) k_cc_roots<<<blocks(V), kThreads, 0, ST>>>(V, W);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_components_keep(int V, int largest, long long min_faces, const uint8_t* workspace, uint8_t* keep, void* stream) {
    if (V < 0 || !workspace || (V > 0 && !keep) || (!largest && min_faces < 0)) return PSDF_ERR_ARG;
    if (V == 0) return PSDF_OK;
    const Ws W = carve(const_cast<uint8_t*>(workspace), V);
    k_cc_keep<<<blocks(V), kThreads, 0, ST>>>(V, largest, min_faces, W, keep);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
