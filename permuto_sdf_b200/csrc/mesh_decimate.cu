// Quadric edge-collapse decimation of an indexed triangle mesh and vertex normals from its faces, sm_90a. Built with -fmad=false:
// every fp64 and fp32 operation is rounded as written, so oracle/decimate.py reproduces the output bit for bit. The rules (quadrics,
// candidates, locks, cost, validity, selection, apply) are stated in include/psdf_b200.h; this file only adds how they are computed.
//
// Vertex -> face CSR (mesh_csr.cuh): k_mesh_degree counts the faces of each vertex, the scan k_mesh_scan_* turns the counts into int64
// offsets, k_mesh_fill places the faces with atomics and k_mesh_sort puts each vertex's list in ascending face order (only begin and the
// normals need the order; a round's CSR is left as filled, every use of it there is order-free). Faces with an index outside [0, V) or a
// repeated vertex are counted by k_mesh_check in begin and never enter the CSR. The compaction scans the faces kept with the same kernels.
//
//   k_dc_lock      a half-edge whose direction is not there once or whose twin is not there once locks both ends   thread per half-edge
//   k_dc_quadric   Q[v] = sum of the area-weighted plane quadrics of v's faces, ascending        thread per vertex
//   k_dc_key       key of every candidate half-edge, best[v] = atomicMin over v's candidates    thread per half-edge
//   k_dc_best2     best2[v] = min of best over v and its neighbours                               thread per vertex
//   k_dc_choose    list += key where key == best2[u] == best2[v]                                 thread per half-edge
//   k_dc_select    the threshold key: the allowed-th smallest of the list (8-bit radix select) when the list is longer   one block
//   k_dc_apply     the chosen collapses with key <= threshold                                     thread per list entry
//   k_dc_compact   faces that no collapse dropped, in order, into the scratch                    thread per face
//   k_dc_copy      the kept faces from the scratch back into the caller's faces                  thread per face
//   k_dc_normals   NV[v] = normalised sum of the cross products of v's faces, ascending           thread per vertex
#include "mesh_csr.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr unsigned long long kNoKey = ~0ull;
// an edge with an end in more faces is no candidate; it bounds the work of a candidate (link condition, flip test) to kMaxFaces^2
constexpr long long kMaxFaces = 64;

// workspace sections in order; the normals use the first five
struct Ws {
    long long* info;          // {faces outside [0, V), faces repeating a vertex, collapses chosen, collapses applied, threshold key}
    long long* off;           // [V + 1] CSR offsets
    int* deg;                 // [V] face count, then the fill cursor
    int* adj;                 // [3F] faces of each vertex
    long long* tiles;         // [tiles + 1] tile sums of the scans
    double* Q;                // [V][10] quadrics
    unsigned long long* best; // [V]
    unsigned long long* best2;// [V]
    uint8_t* lock;            // [V]
    unsigned long long* list; // [V / 2 + 1] chosen keys
    unsigned long long* keys; // [3F] candidate keys; in compaction int64 pos [F + 1], then the kept faces int [3F]
    uint8_t* drop;            // [F]
};

long long carve(void* ws, long long V, long long F, bool decimate, Ws* W) {
    Sections s{static_cast<char*>(ws)};
    Ws w;
    s.take(w.info, kHeaderBytes);
    s.take(w.off, 8 * (V + 1));
    s.take(w.deg, 4 * V);
    s.take(w.adj, 12 * F);
    s.take(w.tiles, 8 * tile_sums(V + 1 > F ? V + 1 : F));
    if (decimate) {
        s.take(w.Q, 80 * V);
        s.take(w.best, 8 * V);
        s.take(w.best2, 8 * V);
        s.take(w.lock, V);
        s.take(w.list, 8 * (V / 2 + 1));
        s.take(w.keys, 24 * F + 8);
        s.take(w.drop, F);
    }
    if (W) *W = w;
    return s.size;
}

// vertex-indexed addresses are formed in 64 bits: 3 v and 10 v overflow int32 long before v does
__device__ __forceinline__ double3 pos64(const float* __restrict__ verts, long long v) {
    return make_double3((double)verts[3 * v], (double)verts[3 * v + 1], (double)verts[3 * v + 2]);
}

__device__ __forceinline__ double3 sub3(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double3 cross3(double3 a, double3 b) {
    return make_double3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ double dot3(double3 a, double3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }

// ---------------------------------------------------------------- locks and quadrics
__device__ __forceinline__ bool follows(int3 t, int u, int v) {
    return (t.x == u && t.y == v) || (t.y == u && t.z == v) || (t.z == u && t.x == v);
}

// (faces holding u -> v, faces holding v -> u, the last of those) of the half-edge u -> v. Both kinds hold u and v, so the list of the
// end with fewer faces is scanned: a half-edge at a vertex of high valence costs the valence of its other end.
struct Twin { int nsame, ntwin, g; };
__device__ Twin find_twin(const Ws& W, const int* __restrict__ faces, int u, int v) {
    Twin r{0, 0, -1};
    const int s = nr_faces(W, v) < nr_faces(W, u) ? v : u;
    for (long long i = W.off[s], e = W.off[s + 1]; i < e; i++) {
        const int h = W.adj[i];
        const int3 t = load_face(faces, h);
        if (follows(t, u, v)) r.nsame++;
        if (follows(t, v, u)) { r.ntwin++; r.g = h; }
    }
    return r;
}

__global__ void __launch_bounds__(kThreads) k_dc_lock(int V, int F, const int* __restrict__ faces, Ws W) {
    const long long c = thread_index();
    if (c >= 3LL * F) return;
    const long long f = c / 3;
    const int k = (int)(c - 3 * f);
    const int3 t = load_face(faces, f);
    if (!valid(t, V)) return;
    const int u = corner(t, k), v = corner(t, k == 2 ? 0 : k + 1);
    const Twin tw = find_twin(W, faces, u, v);
    if (tw.nsame != 1 || tw.ntwin != 1) {
        W.lock[u] = 1;
        W.lock[v] = 1;
    }
}

// the area-weighted plane quadric of face t in fp64, or false for a zero-area face:
// N = (p1 - p0) x (p2 - p0), l = |N|, n = N / l, d = -(n . p0), w = l / 2, q = w * {nx nx, nx ny, nx nz, nx d, ny ny, ny nz, ny d, nz nz,
// nz d, d d}
__device__ bool face_quadric(const float* __restrict__ verts, int3 t, double q[10]) {
    const double3 p0 = pos64(verts, t.x), p1 = pos64(verts, t.y), p2 = pos64(verts, t.z);
    const double3 N = cross3(sub3(p1, p0), sub3(p2, p0));
    const double l = sqrt(dot3(N, N));
    if (!(l > 0.0)) return false;
    const double nx = N.x / l, ny = N.y / l, nz = N.z / l;
    const double d = -((nx * p0.x + ny * p0.y) + nz * p0.z);
    const double w = l * 0.5;
    q[0] = w * (nx * nx); q[1] = w * (nx * ny); q[2] = w * (nx * nz); q[3] = w * (nx * d);
    q[4] = w * (ny * ny); q[5] = w * (ny * nz); q[6] = w * (ny * d);
    q[7] = w * (nz * nz); q[8] = w * (nz * d); q[9] = w * (d * d);
    return true;
}

__global__ void __launch_bounds__(kThreads) k_dc_quadric(int V, const int* __restrict__ faces, const float* __restrict__ verts, Ws W) {
    const long long v = thread_index();
    if (v >= V) return;
    double Q[10];
#pragma unroll
    for (int j = 0; j < 10; j++) Q[j] = 0.0;
    for (long long i = W.off[v], e = W.off[v + 1]; i < e; i++) {
        double q[10];
        if (!face_quadric(verts, load_face(faces, W.adj[i]), q)) continue;
#pragma unroll
        for (int j = 0; j < 10; j++) Q[j] = Q[j] + q[j];
    }
#pragma unroll
    for (int j = 0; j < 10; j++) W.Q[10 * v + j] = Q[j];
}

// ---------------------------------------------------------------- candidates
// v^T Q v with v = (x, y, z, 1), row by row
__device__ __forceinline__ double quadric_error(const double Q[10], double3 p) {
    const double r0 = ((Q[0] * p.x + Q[1] * p.y) + Q[2] * p.z) + Q[3];
    const double r1 = ((Q[1] * p.x + Q[4] * p.y) + Q[5] * p.z) + Q[6];
    const double r2 = ((Q[2] * p.x + Q[5] * p.y) + Q[7] * p.z) + Q[8];
    const double r3 = ((Q[3] * p.x + Q[6] * p.y) + Q[8] * p.z) + Q[9];
    return ((p.x * r0 + p.y * r1) + p.z * r2) + r3;
}

__device__ __forceinline__ double3 to64(float3 p) { return make_double3((double)p.x, (double)p.y, (double)p.z); }

// the position of the unlocked pair (a, b) with Q = Q_a + Q_b and its error
__device__ float3 place(const double Q[10], float3 pa, float3 pb, double& cost) {
    const double c00 = Q[4] * Q[7] - Q[5] * Q[5];
    const double c01 = Q[2] * Q[5] - Q[1] * Q[7];
    const double c02 = Q[1] * Q[5] - Q[4] * Q[2];
    const double c11 = Q[0] * Q[7] - Q[2] * Q[2];
    const double c12 = Q[1] * Q[2] - Q[0] * Q[5];
    const double c22 = Q[0] * Q[4] - Q[1] * Q[1];
    const double det = (Q[0] * c00 + Q[1] * c01) + Q[2] * c02;
    const double tr = (Q[0] + Q[4]) + Q[7];
    if (fabs(det) > 1e-12 * ((tr * tr) * tr)) {
        const double3 x = make_double3(-(((c00 * Q[3] + c01 * Q[6]) + c02 * Q[8]) / det),
                                       -(((c01 * Q[3] + c11 * Q[6]) + c12 * Q[8]) / det),
                                       -(((c02 * Q[3] + c12 * Q[6]) + c22 * Q[8]) / det));
        const double3 a = to64(pa), b = to64(pb);
        const double3 m = make_double3((a.x + b.x) * 0.5, (a.y + b.y) * 0.5, (a.z + b.z) * 0.5);
        const double3 dx = sub3(x, m), e = sub3(b, a);
        if (dot3(dx, dx) <= dot3(e, e)) {
            const float3 p = make_float3((float)x.x, (float)x.y, (float)x.z);
            cost = quadric_error(Q, to64(p));
            return p;
        }
    }
    // near-singular, or the minimiser lies farther from the midpoint than the edge is long: the best of a, b, the midpoint
    const float3 pm = make_float3((pa.x + pb.x) * 0.5f, (pa.y + pb.y) * 0.5f, (pa.z + pb.z) * 0.5f);
    float3 p = pa;
    cost = quadric_error(Q, to64(pa));
    const double cb = quadric_error(Q, to64(pb));
    if (cb < cost) { cost = cb; p = pb; }
    const double cm = quadric_error(Q, to64(pm));
    if (cm < cost) { cost = cm; p = pm; }
    return p;
}

__device__ __forceinline__ bool face_has(int3 t, int x) { return t.x == x || t.y == x || t.z == x; }

// does no face of s other than f and g flip or become degenerate when s moves to p?
__device__ bool faces_hold(const Ws& W, const int* __restrict__ faces, const float* __restrict__ verts, int s, float3 p, int f, int g) {
    const double3 q = to64(p);
    for (long long i = W.off[s], e = W.off[s + 1]; i < e; i++) {
        const int h = W.adj[i];
        if (h == f || h == g) continue;
        const int3 t = load_face(faces, h);
        const double3 p0 = pos64(verts, t.x), p1 = pos64(verts, t.y), p2 = pos64(verts, t.z);
        const double3 n0 = cross3(sub3(p1, p0), sub3(p2, p0));
        const double3 r0 = t.x == s ? q : p0, r1 = t.y == s ? q : p1, r2 = t.z == s ? q : p2;
        const double3 n1 = cross3(sub3(r1, r0), sub3(r2, r0));
        if (!(dot3(n0, n1) > 0.0)) return false;
    }
    return true;
}

struct Collapse { int a, b, f, g; float3 p; double Q[10]; };

// the collapse of candidate half-edge c = 3 f + k -> its key (kNoKey when c is no candidate or fails a check)
__device__ unsigned long long evaluate(const Ws& W, const int* __restrict__ faces, const float* __restrict__ verts, long long c,
                                       Collapse& r) {
    const long long f = c / 3;
    const int k = (int)(c - 3 * f);
    const int3 t = load_face(faces, f);
    const int u = corner(t, k), v = corner(t, k == 2 ? 0 : k + 1), w = corner(t, k == 0 ? 2 : k - 1);
    if (!(u < v) || nr_faces(W, u) > kMaxFaces || nr_faces(W, v) > kMaxFaces) return kNoKey;
    const Twin tw = find_twin(W, faces, u, v);
    if (tw.nsame != 1 || tw.ntwin != 1) return kNoKey;
    const bool lu = W.lock[u] != 0, lv = W.lock[v] != 0;
    if (lu && lv) return kNoKey;
    const int a = lv ? v : u, b = lv ? u : v;
    const int3 tg = load_face(faces, tw.g);
    const int d = tg.x != u && tg.x != v ? tg.x : (tg.y != u && tg.y != v ? tg.y : tg.z);
    if (w == d || nr_faces(W, w) <= 3 || nr_faces(W, d) <= 3) return kNoKey;
    // link condition: b is unlocked, so each of its neighbours follows b in exactly one of its faces
    int common = 0;
    for (long long i = W.off[b], e = W.off[b + 1]; i < e; i++) {
        const int3 h = load_face(faces, W.adj[i]);
        const int x = h.x == b ? h.y : (h.y == b ? h.z : h.x);
        if (x == a) continue;
        for (long long j = W.off[a], ea = W.off[a + 1]; j < ea; j++) {
            if (face_has(load_face(faces, W.adj[j]), x)) { common++; break; }
        }
    }
    if (common != 2) return kNoKey;
#pragma unroll
    for (int j = 0; j < 10; j++) r.Q[j] = W.Q[10LL * a + j] + W.Q[10LL * b + j];
    const float3 pa = load3(verts, a), pb = load3(verts, b);
    double cost;
    if (W.lock[a]) {
        r.p = pa;
        cost = quadric_error(r.Q, to64(pa));
    } else {
        r.p = place(r.Q, pa, pb, cost);
    }
    if (!faces_hold(W, faces, verts, a, r.p, (int)f, tw.g) || !faces_hold(W, faces, verts, b, r.p, (int)f, tw.g)) return kNoKey;
    r.a = a; r.b = b; r.f = (int)f; r.g = tw.g;
    const float cf = (float)(cost > 0.0 ? cost : 0.0);
    return ((unsigned long long)__float_as_uint(cf) << 33) | (unsigned long long)c;
}

__global__ void __launch_bounds__(kThreads) k_dc_key(int F, const int* __restrict__ faces, const float* __restrict__ verts, Ws W) {
    const long long c = thread_index();
    if (c >= 3LL * F) return;
    Collapse r;
    const unsigned long long key = evaluate(W, faces, verts, c, r);
    W.keys[c] = key;
    if (key != kNoKey) {
        atomicMin(W.best + r.a, key);
        atomicMin(W.best + r.b, key);
    }
}

__global__ void __launch_bounds__(kThreads) k_dc_best2(int V, const int* __restrict__ faces, Ws W) {
    const long long v = thread_index();
    if (v >= V) return;
    unsigned long long m = W.best[v];
    for (long long i = W.off[v], e = W.off[v + 1]; i < e; i++) {
        const int3 t = load_face(faces, W.adj[i]);
        m = min(m, min(W.best[t.x], min(W.best[t.y], W.best[t.z])));
    }
    W.best2[v] = m;
}

__global__ void __launch_bounds__(kThreads) k_dc_choose(int F, const int* __restrict__ faces, Ws W) {
    const long long c = thread_index();
    if (c >= 3LL * F) return;
    const unsigned long long key = W.keys[c];
    if (key == kNoKey) return;
    const long long f = c / 3;
    const int k = (int)(c - 3 * f);
    const int3 t = load_face(faces, f);
    const int u = corner(t, k), v = corner(t, k == 2 ? 0 : k + 1);
    if (key == W.best2[u] && key == W.best2[v])
        W.list[atomicAdd(reinterpret_cast<unsigned long long*>(W.info + 2), 1ull)] = key;
}

// threshold = the allowed-th smallest chosen key when more than `allowed` were chosen, else kNoKey (keys are distinct)
__global__ void __launch_bounds__(kTopThreads) k_dc_select(long long allowed, Ws W) {
    __shared__ int hist[256];
    __shared__ unsigned long long prefix;
    __shared__ long long rank;
    const long long n = W.info[2];
    if (n <= allowed) {
        if (threadIdx.x == 0) W.info[4] = (long long)kNoKey;
        return;
    }
    unsigned long long mask = 0;
    if (threadIdx.x == 0) { prefix = 0; rank = allowed; }
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += kTopThreads) hist[i] = 0;
        __syncthreads();
        const unsigned long long pre = prefix;
        for (long long i = threadIdx.x; i < n; i += kTopThreads) {
            const unsigned long long key = W.list[i];
            if ((key & mask) == pre) atomicAdd(hist + ((key >> shift) & 255), 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long r = rank;
            int dgt = 0;
            while (hist[dgt] < r) r -= hist[dgt++];
            rank = r;
            prefix = pre | ((unsigned long long)dgt << shift);
        }
        mask |= 255ull << shift;
        __syncthreads();
    }
    if (threadIdx.x == 0) W.info[4] = (long long)prefix;
}

// chosen collapses never share or neighbour a vertex, so each reads and writes faces, positions and quadrics no other one touches
__global__ void __launch_bounds__(kThreads) k_dc_apply(int V, int* __restrict__ faces, float* __restrict__ verts, Ws W,
                                                       uint8_t* __restrict__ removed) {
    const long long i = thread_index();
    if (i >= W.info[2] || W.list[i] > (unsigned long long)W.info[4]) return;
    Collapse r;
    evaluate(W, faces, verts, (long long)(W.list[i] & ((1ull << 33) - 1)), r);
    verts[3LL * r.a] = r.p.x;
    verts[3LL * r.a + 1] = r.p.y;
    verts[3LL * r.a + 2] = r.p.z;
#pragma unroll
    for (int j = 0; j < 10; j++) W.Q[10LL * r.a + j] = r.Q[j];
    removed[r.b] = 1;
    for (long long j = W.off[r.b], e = W.off[r.b + 1]; j < e; j++) {
        const int h = W.adj[j];
        if (h == r.f || h == r.g) continue;
        for (int q = 0; q < 3; q++)
            if (faces[3LL * h + q] == r.b) faces[3LL * h + q] = r.a;
    }
    W.drop[r.f] = 1;
    W.drop[r.g] = 1;
    atomicAdd(reinterpret_cast<unsigned long long*>(W.info + 3), 1ull);
}

// the scanned value of the compaction: 1 for a face no collapse dropped
struct Kept {
    __device__ __forceinline__ long long operator()(uint8_t drop, long long) const { return drop == 0; }
};

// faces no collapse dropped, in order: pos = exclusive prefix of the kept faces (int64 [F + 1]), the faces go to the scratch behind it
__global__ void __launch_bounds__(kThreads) k_dc_compact(int F, const int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    if (f >= F || W.drop[f]) return;
    const long long* pos = reinterpret_cast<const long long*>(W.keys);
    int* out = reinterpret_cast<int*>(W.keys) + 2 * (F + 1LL) + 3 * pos[f];
    out[0] = faces[3 * f];
    out[1] = faces[3 * f + 1];
    out[2] = faces[3 * f + 2];
}

// the kept faces back from the scratch; rows past the new count keep what they held (the caller reads only the new count)
__global__ void __launch_bounds__(kThreads) k_dc_copy(int F, int* __restrict__ faces, Ws W) {
    const long long f = thread_index();
    const long long* pos = reinterpret_cast<const long long*>(W.keys);
    if (f >= pos[F]) return;
    const int* in = reinterpret_cast<const int*>(W.keys) + 2 * (F + 1LL) + 3 * f;
    faces[3 * f] = in[0];
    faces[3 * f + 1] = in[1];
    faces[3 * f + 2] = in[2];
}

// ---------------------------------------------------------------- normals
__global__ void __launch_bounds__(kThreads) k_dc_normals(int V, const int* __restrict__ faces, const float* __restrict__ verts, Ws W,
                                                         float* __restrict__ normals) {
    const long long v = thread_index();
    if (v >= V) return;
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (long long i = W.off[v], e = W.off[v + 1]; i < e; i++) {
        const int3 t = load_face(faces, W.adj[i]);
        const float3 p0 = load3(verts, t.x), p1 = load3(verts, t.y), p2 = load3(verts, t.z);
        const float ax = p1.x - p0.x, ay = p1.y - p0.y, az = p1.z - p0.z;
        const float bx = p2.x - p0.x, by = p2.y - p0.y, bz = p2.z - p0.z;
        nx = nx + (ay * bz - az * by);
        ny = ny + (az * bx - ax * bz);
        nz = nz + (ax * by - ay * bx);
    }
    const float l = sqrtf((nx * nx + ny * ny) + nz * nz);
    if (l > 0.f) { nx = nx / l; ny = ny / l; nz = nz / l; }
    else { nx = 0.f; ny = 0.f; nz = 0.f; }
    normals[3 * v] = nx;
    normals[3 * v + 1] = ny;
    normals[3 * v + 2] = nz;
}
}  // namespace

extern "C" {

long long psdf_mesh_decimate_workspace_bytes(long long nr_vertices, long long nr_faces) {
    if (nr_vertices < 0 || nr_faces < 0) return PSDF_ERR_ARG;
    if (nr_vertices > kIntMax || nr_faces > kIntMax) return PSDF_ERR_UNSUPPORTED;
    return carve(nullptr, nr_vertices, nr_faces, true, nullptr);
}

long long psdf_mesh_normals_workspace_bytes(long long nr_vertices, long long nr_faces) {
    if (nr_vertices < 0 || nr_faces < 0) return PSDF_ERR_ARG;
    if (nr_vertices > kIntMax || nr_faces > kIntMax) return PSDF_ERR_UNSUPPORTED;
    return carve(nullptr, nr_vertices, nr_faces, false, nullptr);
}

int psdf_mesh_decimate_begin(int V, int F, const float* verts, const int* faces, uint8_t* workspace, uint8_t* removed, void* stream) {
    if (V < 0 || F < 0 || !workspace || (V > 0 && (!verts || !removed)) || (F > 0 && !faces)) return PSDF_ERR_ARG;
    Ws W;
    carve(workspace, V, F, true, &W);
    cudaMemsetAsync(W.info, 0, kHeaderBytes, ST);
    if (V > 0) {
        cudaMemsetAsync(removed, 0, (size_t)V, ST);
        cudaMemsetAsync(W.lock, 0, (size_t)V, ST);
    }
    if (F > 0) k_mesh_check<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
    build_csr(V, F, faces, W, true, ST);
    if (F > 0) k_dc_lock<<<blocks(3LL * F), kThreads, 0, ST>>>(V, F, faces, W);
    if (V > 0) k_dc_quadric<<<blocks(V), kThreads, 0, ST>>>(V, faces, verts, W);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_decimate_round(int V, int F0, int F, long long allowed, float* verts, int* faces, uint8_t* workspace, uint8_t* removed,
                             void* stream) {
    if (V < 0 || F < 0 || F > F0 || allowed < 0 || !workspace || (V > 0 && (!verts || !removed)) || (F > 0 && !faces))
        return PSDF_ERR_ARG;
    Ws W;
    carve(workspace, V, F0, true, &W);
    cudaMemsetAsync(W.info + 2, 0, 3 * sizeof(long long), ST);
    if (F == 0 || allowed == 0) return PSDF_OK;
    build_csr(V, F, faces, W, false, ST);
    cudaMemsetAsync(W.best, 0xff, 8 * (size_t)V, ST);
    cudaMemsetAsync(W.drop, 0, (size_t)F, ST);
    k_dc_key<<<blocks(3LL * F), kThreads, 0, ST>>>(F, faces, verts, W);
    k_dc_best2<<<blocks(V), kThreads, 0, ST>>>(V, faces, W);
    k_dc_choose<<<blocks(3LL * F), kThreads, 0, ST>>>(F, faces, W);
    k_dc_select<<<1, kTopThreads, 0, ST>>>(allowed, W);
    k_dc_apply<<<blocks(V / 2 + 1), kThreads, 0, ST>>>(V, faces, verts, W, removed);
    long long* pos = reinterpret_cast<long long*>(W.keys);
    scan<Kept>(W.drop, F, W.tiles, pos, ST);
    k_dc_compact<<<blocks(F), kThreads, 0, ST>>>(F, faces, W);
    k_dc_copy<<<blocks(F), kThreads, 0, ST>>>(F, faces, W);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_normals(int V, int F, const float* verts, const int* faces, uint8_t* workspace, float* normals, void* stream) {
    if (V < 0 || F < 0 || !workspace || (V > 0 && (!verts || !normals)) || (F > 0 && !faces)) return PSDF_ERR_ARG;
    Ws W;
    carve(workspace, V, F, false, &W);
    cudaMemsetAsync(W.info, 0, kHeaderBytes, ST);
    if (F > 0) k_mesh_check<<<blocks(F), kThreads, 0, ST>>>(V, F, faces, W);
    build_csr(V, F, faces, W, true, ST);
    if (V > 0) k_dc_normals<<<blocks(V), kThreads, 0, ST>>>(V, faces, verts, W, normals);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
