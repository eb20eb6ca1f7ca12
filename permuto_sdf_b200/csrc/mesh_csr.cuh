// The vertex -> face CSR of an indexed triangle mesh and what builds it, shared by mesh_decimate.cu, mesh_distance.cu (pseudonormals)
// and mesh_subdivide.cu.
//
// A unit lays out its own workspace Ws with Sections. Every such Ws holds at least
//   long long* info;   int64 header: info[0] = faces with an index outside [0, V), info[1] = faces that repeat a vertex
//   long long* off;    [V + 1] CSR offsets
//   int* deg;          [V] face count, then the fill cursor
// and the kernels here are templates on it. build_csr also needs
//   int* adj;          [3F] faces of each vertex
//   long long* tiles;  scan tile sums of at least tile_sums(V) entries
// and fills the face lists; a unit that fills more than the lists (mesh_subdivide.cu) launches k_mesh_degree and the scan itself. The
// offsets come from an exclusive int64 scan (k_mesh_scan_tiles, k_mesh_scan_top, k_mesh_scan_out) of op(a[i], i) over an array a: Count
// here, and what a unit scans besides.
//
//   k_mesh_check      counts faces outside [0, V) and faces that repeat a vertex into info[0], info[1]   thread per face
//   k_mesh_degree     deg[v] += 1 for the three corners of every valid face                             thread per face
//   k_mesh_scan_*     exclusive prefix of op(a[i], i) over [0, n) and its total                          tile / one block / tile
//   k_mesh_fill       adj[off[v] + cursor] = f for the three corners of every valid face                thread per face
//   k_mesh_sort       heap sort of each vertex's face list                                              thread per vertex
#pragma once
#include "common.cuh"

#define ST ((cudaStream_t)stream)

namespace {
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kThreads = 256;
constexpr int kTileItems = 8;                                 // scan: elements per thread in a tile
constexpr long long kTile = (long long)kThreads * kTileItems;
constexpr int kTopThreads = 1024;
constexpr long long kHeaderBytes = 256;
constexpr long long kIntMax = 0x7fffffffLL;

long long align256(long long n) { return (n + 255) & ~255LL; }
unsigned blocks(long long n) { return (unsigned)(n > 0 ? psdf::div_up(n, kThreads) : 1); }
// entries of the tile sums of a scan of up to n values: one per tile and the total
long long tile_sums(long long n) { return (n + kTile - 1) / kTile + 1; }

// workspace sections one after another, each padded to 256 bytes; with a null base only their size is added up
struct Sections {
    char* base;
    long long size = 0;
    template <class T> void take(T*& p, long long bytes) {
        p = base ? reinterpret_cast<T*>(base + size) : nullptr;
        size += align256(bytes);
    }
};

__device__ __forceinline__ long long thread_index() { return (long long)blockIdx.x * kThreads + threadIdx.x; }

__device__ __forceinline__ int3 load_face(const int* __restrict__ faces, long long f) {
    const int* p = faces + 3 * f;
    return make_int3(p[0], p[1], p[2]);
}

__device__ __forceinline__ int corner(int3 t, int k) { return k == 0 ? t.x : (k == 1 ? t.y : t.z); }

__device__ __forceinline__ bool in_range(int3 t, int V) {
    return (unsigned)t.x < (unsigned)V && (unsigned)t.y < (unsigned)V && (unsigned)t.z < (unsigned)V;
}
__device__ __forceinline__ bool distinct(int3 t) { return t.x != t.y && t.y != t.z && t.z != t.x; }
__device__ __forceinline__ bool valid(int3 t, int V) { return in_range(t, V) && distinct(t); }

// vertex-indexed addresses are formed in 64 bits: 3 v overflows int32 long before v does
__device__ __forceinline__ float3 load3(const float* __restrict__ verts, long long v) {
    return make_float3(verts[3 * v], verts[3 * v + 1], verts[3 * v + 2]);
}

template <class Ws> __device__ __forceinline__ long long nr_faces(const Ws& W, int v) { return W.off[v + 1] - W.off[v]; }

// ---------------------------------------------------------------- checks and degrees
template <class Ws>
__global__ void __launch_bounds__(kThreads) k_mesh_check(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    bool out = false, rep = false;
    if (f < F) {
        const int3 t = load_face(faces, f);
        out = !in_range(t, V);
        rep = !out && !distinct(t);
    }
    const unsigned mo = __ballot_sync(kFullMask, out), mr = __ballot_sync(kFullMask, rep);
    if ((threadIdx.x & 31) == 0) {
        if (mo) atomicAdd(reinterpret_cast<unsigned long long*>(W.info), (unsigned long long)__popc(mo));
        if (mr) atomicAdd(reinterpret_cast<unsigned long long*>(W.info + 1), (unsigned long long)__popc(mr));
    }
}

template <class Ws>
__global__ void __launch_bounds__(kThreads) k_mesh_degree(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    if (f >= F) return;
    const int3 t = load_face(faces, f);
    if (!valid(t, V)) return;
    atomicAdd(W.deg + t.x, 1);
    atomicAdd(W.deg + t.y, 1);
    atomicAdd(W.deg + t.z, 1);
}

// ---------------------------------------------------------------- exclusive int64 scan
// the scanned value of a count array
struct Count {
    __device__ __forceinline__ long long operator()(int x, long long) const { return x; }
};

// inclusive block prefix of x over kThreads threads -> (inclusive value, block total)
__device__ __forceinline__ long long block_inclusive(long long x, long long& total) {
    __shared__ long long sh[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(kFullMask, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    if (warp == 0) {
        long long w = lane < kThreads / 32 ? sh[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(kFullMask, w, o);
            if (lane >= o) w += y;
        }
        if (lane < kThreads / 32) sh[lane] = w;
    }
    __syncthreads();
    const long long r = x + (warp ? sh[warp - 1] : 0);
    total = sh[kThreads / 32 - 1];
    __syncthreads();
    return r;
}

template <class Op, class T> __device__ __forceinline__ long long scan_value(const T* __restrict__ a, long long n, long long i) {
    return i < n ? Op()(a[i], i) : 0;
}

// tile sums: tiles[b] = the sum of the values of tile b
template <class Op, class T>
__global__ void __launch_bounds__(kThreads) k_mesh_scan_tiles(const T* __restrict__ a, long long n, long long* __restrict__ tiles) {
    const long long b0 = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kTileItems;
    long long s = 0;
    for (int j = 0; j < kTileItems; j++) s += scan_value<Op>(a, n, b0 + j);
    long long total;
    block_inclusive(s, total);
    if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

// exclusive prefix of the tile sums in place, in chunks of kTopThreads; tiles[ntiles] = the total
__global__ void __launch_bounds__(kTopThreads) k_mesh_scan_top(long long* __restrict__ tiles, long long ntiles) {
    __shared__ long long sh[kTopThreads / 32];
    __shared__ long long carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (long long c0 = 0; c0 < ntiles; c0 += kTopThreads) {
        const long long i = c0 + threadIdx.x;
        const long long v = i < ntiles ? tiles[i] : 0;
        long long x = v;
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(kFullMask, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) sh[warp] = x;
        __syncthreads();
        if (warp == 0) {
            long long w = sh[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const long long y = __shfl_up_sync(kFullMask, w, o);
                if (lane >= o) w += y;
            }
            sh[lane] = w;
        }
        __syncthreads();
        const long long base = carry;
        if (i < ntiles) tiles[i] = base + x - v + (warp ? sh[warp - 1] : 0);
        __syncthreads();
        if (threadIdx.x == 0) carry = base + sh[kTopThreads / 32 - 1];
        __syncthreads();
    }
    if (threadIdx.x == 0) tiles[ntiles] = carry;
}

// out[i] = exclusive prefix, out[n] = total. Bound by memory: 8 blocks per SM (32 registers) keep more loads in flight than the 40
// registers ptxas would take for the count array
template <class Op, class T>
__global__ void __launch_bounds__(kThreads, 8) k_mesh_scan_out(const T* __restrict__ a, long long n, const long long* __restrict__ tiles,
                                                               long long ntiles, long long* __restrict__ out) {
    const long long b0 = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kTileItems;
    long long v[kTileItems], s = 0;
    for (int j = 0; j < kTileItems; j++) {
        v[j] = scan_value<Op>(a, n, b0 + j);
        s += v[j];
    }
    long long total;
    long long run = block_inclusive(s, total) - s + tiles[blockIdx.x];
    for (int j = 0; j < kTileItems; j++) {
        if (b0 + j < n) out[b0 + j] = run;
        run += v[j];
    }
    if (threadIdx.x == 0 && blockIdx.x == 0) out[n] = tiles[ntiles];
}

// exclusive scan of op(a[i], i) over [0, n) into out [n + 1]; tiles holds tile_sums(n) entries
template <class Op, class T>
void scan(const T* a, long long n, long long* tiles, long long* out, cudaStream_t s) {
    const long long nt = (n + kTile - 1) / kTile;
    if (nt > 0) k_mesh_scan_tiles<Op><<<(unsigned)nt, kThreads, 0, s>>>(a, n, tiles);
    k_mesh_scan_top<<<1, kTopThreads, 0, s>>>(tiles, nt);
    if (nt > 0) k_mesh_scan_out<Op><<<(unsigned)nt, kThreads, 0, s>>>(a, n, tiles, nt, out);
    else cudaMemsetAsync(out, 0, sizeof(long long), s);
}

// ---------------------------------------------------------------- sorting a vertex's list
__device__ void sift_down(int* a, long long i, long long n) {
    const int x = a[i];
    for (long long c = 2 * i + 1; c < n; c = 2 * i + 1) {
        if (c + 1 < n && a[c + 1] > a[c]) c++;
        if (a[c] <= x) break;
        a[i] = a[c];
        i = c;
    }
    a[i] = x;
}

// heap sort of a[0, n) in ascending order, O(n log n) for a vertex of any valence (a fan of 10^5 faces sorts in about 2 * 10^6 steps)
__device__ __forceinline__ void heap_sort(int* a, long long n) {
    for (long long i = n / 2 - 1; i >= 0; i--) sift_down(a, i, n);
    for (long long e = n - 1; e > 0; e--) {
        const int x = a[0];
        a[0] = a[e];
        a[e] = x;
        sift_down(a, 0, e);
    }
}

// ---------------------------------------------------------------- the CSR
template <class Ws>
__global__ void __launch_bounds__(kThreads) k_mesh_fill(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    if (f >= F) return;
    const int3 t = load_face(faces, f);
    if (!valid(t, V)) return;
    W.adj[W.off[t.x] + atomicAdd(W.deg + t.x, 1)] = (int)f;
    W.adj[W.off[t.y] + atomicAdd(W.deg + t.y, 1)] = (int)f;
    W.adj[W.off[t.z] + atomicAdd(W.deg + t.z, 1)] = (int)f;
}

template <class Ws> __global__ void __launch_bounds__(kThreads) k_mesh_sort(int V, Ws W) {
    const long long v = thread_index();
    if (v >= V) return;
    heap_sort(W.adj + W.off[v], W.off[v + 1] - W.off[v]);
}

// the CSR of the valid faces (deg and off rebuilt); sorted: each vertex's list in ascending face order, else in fill order
template <class Ws> void build_csr(int V, int F, const int* faces, const Ws& W, bool sorted, cudaStream_t s) {
    cudaMemsetAsync(W.deg, 0, 4 * (size_t)V, s);
    if (F > 0) k_mesh_degree<<<blocks(F), kThreads, 0, s>>>(V, F, faces, W);
    scan<Count>(W.deg, V, W.tiles, W.off, s);
    cudaMemsetAsync(W.deg, 0, 4 * (size_t)V, s);
    if (F > 0) k_mesh_fill<<<blocks(F), kThreads, 0, s>>>(V, F, faces, W);
    if (sorted && V > 0) k_mesh_sort<<<blocks(V), kThreads, 0, s>>>(V, W);
}
}  // namespace
