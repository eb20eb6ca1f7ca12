// Marching cubes over a volume streamed in slabs of slices along axis 0, sm_90a. Replaces skimage.measure.marching_cubes as
// extract_mesh_from_sdf_model calls it (permuto_sdf_py/utils/sdf_utils.py:280-283) on a dense host volume.
//
// Volume [N0, N1, N2], axis 0 = x. A corner is inside when value < threshold (NaN and equality: outside). One vertex per crossing grid
// edge at corner + t along the edge axis, t = (threshold - f_lo) / (f_hi - f_lo) rounded per operation (the unit builds with -fmad=false,
// and every operation is written out anyway).
//
// Canonical order, independent of the slab split: vertices slice by slice, for slice i its crossing axis-1 edges, then its axis-2 edges
// (both row-major in (j, k)), then the crossing axis-0 edges between slices i and i + 1; faces cell by cell, row-major in (i, j, k), and in
// table order within a cell. A slab of S cell slices reads S + 1 slices; its edges, in that order, are
//   [in-plane(0), axis-0(0), in-plane(1), axis-0(1), ..., in-plane(S-1), axis-0(S-1), in-plane(S)]
// and their exclusive prefix count plus the vertices of earlier slabs is their global id. The in-plane edges of slice S are the first
// edges of the next slab, so they get the same ids there; they are emitted by the next slab (or by this one when slice S is the last).
// Ids and positions come from prefix sums over fixed tiles, not from atomics: the result is the same bits on every run.
//
//   k_mc_table      the triangle table (generated on the host at load, below) into the workspace             1 block
//   k_mc_count      crossings per edge tile and triangles per cell tile                                       1 launch
//   k_mc_scan       exclusive prefix of the tile counts, the slab's counts                                    1 block
//   k_mc_vertices   edge ids of the slab, vertices of the emitted edges                                       1 launch
//   k_mc_faces      triangles of the slab's cells                                                             1 launch
#include "common.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kThreads = 256;
constexpr int kRounds = 8;
constexpr int kTile = kThreads * kRounds;        // edges or cells per block of the count and emit kernels
constexpr int kMaxTri = 10;                      // triangles of a cell: crossing edges (<= 12) - 2 per loop
constexpr int kScanThreads = 1024;
constexpr long long kIntMax = 0x7fffffffLL;
#define ST ((cudaStream_t)stream)

struct McTable {
    uint8_t ntri[256];
    int8_t tri[256][3 * kMaxTri];                // edge numbers 4 a + m of the cell, three per triangle
};
constexpr size_t kTableBytes = 8192;
static_assert(sizeof(McTable) <= kTableBytes, "table area");

// ---------------------------------------------------------------------------------------------- table, generated at load
// Corner c at (c & 1, c >> 1 & 1, c >> 2 & 1). Edge 4 a + m along axis a; bits 0 and 1 of m are the offsets along the other two axes,
// lower axis first. On each cube face the crossing edges are joined by segments; a face with 4 crossings cuts off its two inside
// corners, so the two cells of a face always agree. Every crossing edge lies on two faces and ends one segment on each: the segments
// close into loops. Loops are taken in the order of their smallest edge, start there, run so that the right-hand normal points from
// inside to outside, and are fanned from their first edge.
int corner_of(const int p[3]) { return p[0] | p[1] << 1 | p[2] << 2; }

void other_axes(int a, int& o0, int& o1) {
    o0 = a == 0 ? 1 : 0;
    o1 = a == 2 ? 1 : 2;
}

int edge_between(int c0, int c1) {          // corners that differ along one axis
    const int d = c0 ^ c1;
    const int a = d == 1 ? 0 : (d == 2 ? 1 : 2);
    const int lo = c0 < c1 ? c0 : c1;
    int o0, o1;
    other_axes(a, o0, o1);
    return 4 * a + ((lo >> o0 & 1) | (lo >> o1 & 1) << 1);
}

void edge_mid2(int e, int v[3]) {           // twice the edge midpoint
    const int a = e >> 2, m = e & 3;
    int o0, o1;
    other_axes(a, o0, o1);
    v[a] = 1;
    v[o0] = 2 * (m & 1);
    v[o1] = 2 * (m >> 1 & 1);
}

McTable make_table() {
    McTable T = {};
    for (int cfg = 0; cfg < 256; cfg++) {
        int seg_a[12], seg_b[12], seg_axis[12], seg_side[12], seg_ref[12], nseg = 0;
        for (int a = 0; a < 3; a++)
            for (int s = 0; s < 2; s++) {
                int u, v;
                other_axes(a, u, v);
                int q[4], in[4], E[4];
                const int cyc[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}};
                for (int k = 0; k < 4; k++) {
                    int p[3];
                    p[a] = s; p[u] = cyc[k][0]; p[v] = cyc[k][1];
                    q[k] = corner_of(p);
                    in[k] = cfg >> q[k] & 1;
                }
                int nx = 0, xk[4];
                for (int k = 0; k < 4; k++) {
                    E[k] = edge_between(q[k], q[(k + 1) & 3]);
                    if (in[k] != in[(k + 1) & 3]) xk[nx++] = k;
                }
                auto add = [&](int ea, int eb, int ref) {
                    seg_a[nseg] = ea; seg_b[nseg] = eb; seg_axis[nseg] = a; seg_side[nseg] = s; seg_ref[nseg] = ref; nseg++;
                };
                if (nx == 2) {
                    int ref = 0;
                    for (int k = 3; k >= 0; k--)
                        if (in[k]) ref = q[k];
                    add(E[xk[0]], E[xk[1]], ref);
                } else if (nx == 4) {
                    for (int k = 0; k < 4; k++)
                        if (in[k]) add(E[(k + 3) & 3], E[k], q[k]);
                }
            }
        // each crossing edge: its two segments
        int nb[12][2], ns[12][2], deg[12] = {0};
        for (int i = 0; i < nseg; i++) {
            nb[seg_a[i]][deg[seg_a[i]]] = seg_b[i]; ns[seg_a[i]][deg[seg_a[i]]++] = i;
            nb[seg_b[i]][deg[seg_b[i]]] = seg_a[i]; ns[seg_b[i]][deg[seg_b[i]]++] = i;
        }
        bool seen[12] = {false};
        int ntri = 0;
        for (int e0 = 0; e0 < 12; e0++) {
            if (!deg[e0] || seen[e0]) continue;
            // direction: the segment e0 -> nb[e0][0] keeps its inside corner on the right, seen from outside the cube
            const int sg = ns[e0][0];
            int m0[3], m1[3], c[3], d[3], r[3];
            edge_mid2(e0, m0);
            edge_mid2(nb[e0][0], m1);
            const int ref = seg_ref[sg];
            c[0] = 2 * (ref & 1); c[1] = 2 * (ref >> 1 & 1); c[2] = 2 * (ref >> 2 & 1);
            for (int k = 0; k < 3; k++) { d[k] = m1[k] - m0[k]; r[k] = c[k] - m0[k]; }
            const int cr[3] = {d[1] * r[2] - d[2] * r[1], d[2] * r[0] - d[0] * r[2], d[0] * r[1] - d[1] * r[0]};
            const int side = cr[seg_axis[sg]] * (2 * seg_side[sg] - 1);
            int loop[12], L = 0, prev = e0, cur = side < 0 ? nb[e0][0] : nb[e0][1];
            loop[L++] = e0;
            seen[e0] = true;
            while (cur != e0) {
                loop[L++] = cur;
                seen[cur] = true;
                const int next = nb[cur][0] == prev ? nb[cur][1] : nb[cur][0];
                prev = cur;
                cur = next;
            }
            for (int k = 1; k + 1 < L; k++) {
                T.tri[cfg][3 * ntri] = (int8_t)loop[0];
                T.tri[cfg][3 * ntri + 1] = (int8_t)loop[k];
                T.tri[cfg][3 * ntri + 2] = (int8_t)loop[k + 1];
                ntri++;
            }
        }
        T.ntri[cfg] = (uint8_t)ntri;
    }
    return T;
}

const McTable g_table = make_table();

// ---------------------------------------------------------------------------------------------- slab geometry
struct Slab {
    const float* vol;          // [S + 1, N1, N2], slice 0 = global slice i0
    int S, N1, N2, i0, last;
    float thr;
    int E1, Ein, B;            // axis-1 edges of a slice, in-plane edges of a slice, edges per slice step (in-plane + axis 0)
    int ne_main, ne;           // S * B: edges up to the last slice; all edges of the slab (+ in-plane of slice S)
    int nb_main, nb_edge;      // edge tiles: [0, nb_main) cover [0, ne_main), the rest cover the in-plane edges of slice S
    int ncell, nb_cell;
};

Slab make_slab(const float* vol, int S, int N1, int N2, int i0, int last, float thr) {
    Slab L;
    L.vol = vol; L.S = S; L.N1 = N1; L.N2 = N2; L.i0 = i0; L.last = last; L.thr = thr;
    L.E1 = (N1 - 1) * N2;
    L.Ein = L.E1 + N1 * (N2 - 1);
    L.B = L.Ein + N1 * N2;
    L.ne_main = S * L.B;
    L.ne = L.ne_main + L.Ein;
    L.nb_main = div_up(L.ne_main, kTile);
    L.nb_edge = L.nb_main + div_up(L.Ein, kTile);
    L.ncell = S * (N1 - 1) * (N2 - 1);
    L.nb_cell = div_up(L.ncell, kTile);
    return L;
}

// limits of one slab: every slab-local index and count fits in int32
bool slab_ok(int S, int N1, int N2) {
    if (S < 1 || N1 < 2 || N2 < 2) return false;
    const long long P = (long long)N1 * N2;
    const long long Ein = 2 * P - N1 - N2;
    const long long ne = (long long)S * (Ein + P) + Ein;
    const long long cells = (long long)S * (N1 - 1) * (N2 - 1);
    return ne <= kIntMax - kTile && cells * kMaxTri <= kIntMax - kTile;
}

struct EdgeRef { int s, axis, j, k; };

__device__ __forceinline__ bool inside(float v, float thr) { return v < thr; }

__device__ __forceinline__ const float* at(const Slab& L, int s, int j, int k) {
    return L.vol + ((long long)s * L.N1 + j) * L.N2 + k;
}

// slab edge e -> (slice, axis, j, k) and its two values (lower-index end first)
__device__ __forceinline__ EdgeRef edge_ref(const Slab& L, int e, float& lo, float& hi) {
    EdgeRef R;
    R.s = e / L.B;
    int r = e - R.s * L.B;
    if (r < L.E1) {
        R.axis = 1; R.j = r / L.N2; R.k = r - R.j * L.N2;
        lo = __ldg(at(L, R.s, R.j, R.k)); hi = __ldg(at(L, R.s, R.j + 1, R.k));
    } else if (r < L.Ein) {
        r -= L.E1;
        R.axis = 2; R.j = r / (L.N2 - 1); R.k = r - R.j * (L.N2 - 1);
        lo = __ldg(at(L, R.s, R.j, R.k)); hi = __ldg(at(L, R.s, R.j, R.k + 1));
    } else {
        r -= L.Ein;
        R.axis = 0; R.j = r / L.N2; R.k = r - R.j * L.N2;
        lo = __ldg(at(L, R.s, R.j, R.k)); hi = __ldg(at(L, R.s + 1, R.j, R.k));
    }
    return R;
}

// edge tile b -> [begin, end) of slab edges
__device__ __forceinline__ void edge_tile(const Slab& L, int b, int& begin, int& end) {
    if (b < L.nb_main) {
        begin = b * kTile;
        end = min(begin + kTile, L.ne_main);
    } else {
        begin = L.ne_main + (b - L.nb_main) * kTile;
        end = min(begin + kTile, L.ne);
    }
}

__device__ __forceinline__ int cube_of(const Slab& L, int c, int& s, int& j, int& k) {
    const int per = (L.N1 - 1) * (L.N2 - 1);
    s = c / per;
    const int r = c - s * per;
    j = r / (L.N2 - 1);
    k = r - j * (L.N2 - 1);
    int cube = 0;
#pragma unroll
    for (int q = 0; q < 8; q++)
        cube |= (int)inside(__ldg(at(L, s + (q & 1), j + (q >> 1 & 1), k + (q >> 2 & 1))), L.thr) << q;
    return cube;
}

// slab edge index of edge 4 a + m of cell (s, j, k)
__device__ __forceinline__ int cell_edge(const Slab& L, int s, int j, int k, int e) {
    const int a = e >> 2, b0 = e & 1, b1 = e >> 1 & 1;
    if (a == 0) return s * L.B + L.Ein + (j + b0) * L.N2 + (k + b1);
    if (a == 1) return (s + b0) * L.B + j * L.N2 + (k + b1);
    return (s + b0) * L.B + L.E1 + (j + b1) * (L.N2 - 1) + k;
}

// exclusive prefix of v over the block in thread order; *total = block sum. Two __syncthreads; `sh` holds kThreads / 32 ints.
__device__ __forceinline__ int block_exclusive(int v, int* sh, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(kFullMask, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    int before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; w++) {
        const int t = sh[w];
        before += w < warp ? t : 0;
        total += t;
    }
    __syncthreads();
    return before + x - v;
}

// ---------------------------------------------------------------------------------------------- kernels
__global__ void k_mc_table(McTable T, McTable* out) {
    const int c = threadIdx.x;
    out->ntri[c] = T.ntri[c];
    for (int q = 0; q < 3 * kMaxTri; q++) out->tri[c][q] = T.tri[c][q];
}

// tile counts: blocks [0, nb_edge) count crossing edges, blocks [nb_edge, nb_edge + nb_cell) count triangles
__global__ void __launch_bounds__(kThreads) k_mc_count(Slab L, const McTable* __restrict__ tab, int* __restrict__ tiles) {
    __shared__ int sh[kThreads / 32];
    int n = 0;
    if ((int)blockIdx.x < L.nb_edge) {
        int begin, end;
        edge_tile(L, blockIdx.x, begin, end);
        for (int e = begin + threadIdx.x; e < end; e += kThreads) {
            float lo, hi;
            edge_ref(L, e, lo, hi);
            n += inside(lo, L.thr) != inside(hi, L.thr);
        }
    } else {
        const int begin = (blockIdx.x - L.nb_edge) * kTile, end = min(begin + kTile, L.ncell);
        for (int c = begin + threadIdx.x; c < end; c += kThreads) {
            int s, j, k;
            n += __ldg(&tab->ntri[cube_of(L, c, s, j, k)]);
        }
    }
    int total;
    block_exclusive(n, sh, total);
    if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

// exclusive prefix over one run of tile counts, in place; -> the run's total. Serial chunks per thread, then a block prefix.
__device__ int scan_run(int* a, int n) {
    __shared__ int sh[kScanThreads / 32];
    __shared__ int tot;
    const int per = (n + kScanThreads - 1) / kScanThreads;
    const int b = threadIdx.x * per, e = min(b + per, n);
    int sum = 0;
    for (int i = b; i < e; i++) sum += a[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = sum;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(kFullMask, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = sh[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(kFullMask, w, o);
            if (lane >= o) w += y;
        }
        sh[lane] = w;
        if (lane == 31) tot = w;
    }
    __syncthreads();
    int run = (warp ? sh[warp - 1] : 0) + x - sum;
    for (int i = b; i < e; i++) {
        const int v = a[i];
        a[i] = run;
        run += v;
    }
    const int t = tot;
    __syncthreads();
    return t;
}

// counts [3] = {vertices this slab emits, triangles of its cells, crossing edges of the slab including the in-plane edges of slice S}
__global__ void __launch_bounds__(kScanThreads) k_mc_scan(Slab L, int* __restrict__ tiles, long long* __restrict__ counts) {
    const int ne = scan_run(tiles, L.nb_edge);
    const int nf = scan_run(tiles + L.nb_edge, L.nb_cell);
    if (threadIdx.x == 0) {
        counts[0] = L.last ? ne : tiles[L.nb_main];
        counts[1] = nf;
        counts[2] = ne;
    }
}

struct Affine { float div, mul, off; };     // output coordinate = (index coordinate / div) * mul + off

__device__ __forceinline__ float affine(float x, const Affine& A) { return __fadd_rn(__fmul_rn(__fdiv_rn(x, A.div), A.mul), A.off); }

// ids [ne]: global vertex id of every crossing edge of the slab; verts [counts[0], 3]: the emitted vertices
__global__ void __launch_bounds__(kThreads) k_mc_vertices(Slab L, long long vbase, Affine A, const int* __restrict__ tiles, int* __restrict__ ids,
                                                          float* __restrict__ verts) {
    __shared__ int sh[kThreads / 32];
    int begin, end;
    edge_tile(L, blockIdx.x, begin, end);
    int pos = tiles[blockIdx.x];
    for (int r = 0; r < kRounds; r++) {
        const int e = begin + r * kThreads + threadIdx.x;
        float lo = 0.f, hi = 0.f;
        EdgeRef R = {0, 0, 0, 0};
        bool x = false;
        if (e < end) {
            R = edge_ref(L, e, lo, hi);
            x = inside(lo, L.thr) != inside(hi, L.thr);
        }
        int total;
        const int p = pos + block_exclusive((int)x, sh, total);
        if (x) {
            ids[e] = (int)(vbase + p);
            if (e < L.ne_main || L.last) {
                const float t = __fdiv_rn(__fsub_rn(L.thr, lo), __fsub_rn(hi, lo));
                float c[3] = {(float)(L.i0 + R.s), (float)R.j, (float)R.k};
                c[R.axis] = __fadd_rn(c[R.axis], t);
                float* o = verts + 3 * (long long)p;
                o[0] = affine(c[0], A); o[1] = affine(c[1], A); o[2] = affine(c[2], A);
            }
        }
        pos += total;
    }
}

// faces [counts[1], 3]: slab-local triangle position from the tile prefix, vertex ids from `ids`
__global__ void __launch_bounds__(kThreads) k_mc_faces(Slab L, const McTable* __restrict__ tab, const int* __restrict__ tiles,
                                                       const int* __restrict__ ids, int* __restrict__ faces) {
    __shared__ int sh[kThreads / 32];
    const int begin = blockIdx.x * kTile;
    int pos = tiles[L.nb_edge + blockIdx.x];
    for (int r = 0; r < kRounds; r++) {
        const int c = begin + r * kThreads + threadIdx.x;
        int s = 0, j = 0, k = 0, cube = 0, n = 0;
        if (c < L.ncell) {
            cube = cube_of(L, c, s, j, k);
            n = __ldg(&tab->ntri[cube]);
        }
        int total;
        const int p = pos + block_exclusive(n, sh, total);
        for (int q = 0; q < 3 * n; q++)
            faces[3 * (long long)p + q] = __ldg(&ids[cell_edge(L, s, j, k, __ldg(&tab->tri[cube][q]))]);
        pos += total;
    }
}

struct Workspace { McTable* table; int* tiles; int* ids; };

Workspace carve(void* ws, const Slab& L) {
    Workspace W;
    char* p = static_cast<char*>(ws);
    W.table = reinterpret_cast<McTable*>(p);
    W.tiles = reinterpret_cast<int*>(p + kTableBytes);
    W.ids = W.tiles + ((L.nb_edge + L.nb_cell + 63) / 64) * 64;
    return W;
}
}  // namespace

extern "C" {

long long psdf_marching_cubes_workspace_bytes(int S, int N1, int N2) {
    if (!slab_ok(S, N1, N2)) return PSDF_ERR_UNSUPPORTED;
    const Slab L = make_slab(nullptr, S, N1, N2, 0, 0, 0.f);
    return (long long)kTableBytes + 4LL * ((L.nb_edge + L.nb_cell + 63) / 64) * 64 + 4LL * L.ne;
}

int psdf_marching_cubes_count(int S, int N1, int N2, int i0, int last, float threshold, const float* vol, uint8_t* workspace, long long* counts,
                              void* stream) {
    if (!vol || !workspace || !counts || i0 < 0) return PSDF_ERR_ARG;
    if (!slab_ok(S, N1, N2)) return PSDF_ERR_UNSUPPORTED;
    const Slab L = make_slab(vol, S, N1, N2, i0, last, threshold);
    const Workspace W = carve(workspace, L);
    k_mc_table<<<1, 256, 0, ST>>>(g_table, W.table);
    k_mc_count<<<L.nb_edge + L.nb_cell, kThreads, 0, ST>>>(L, W.table, W.tiles);
    k_mc_scan<<<1, kScanThreads, 0, ST>>>(L, W.tiles, counts);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_marching_cubes_emit(int S, int N1, int N2, int i0, int last, float threshold, const float* vol, long long vertex_base,
                             const float affine_div_mul_off[3], uint8_t* workspace, float* verts, int* faces, void* stream) {
    if (!vol || !workspace || !affine_div_mul_off || i0 < 0 || vertex_base < 0) return PSDF_ERR_ARG;
    if (!slab_ok(S, N1, N2)) return PSDF_ERR_UNSUPPORTED;
    const Slab L = make_slab(vol, S, N1, N2, i0, last, threshold);
    const Workspace W = carve(workspace, L);
    const Affine A = {affine_div_mul_off[0], affine_div_mul_off[1], affine_div_mul_off[2]};
    k_mc_vertices<<<L.nb_edge, kThreads, 0, ST>>>(L, vertex_base, A, W.tiles, W.ids, verts);
    k_mc_faces<<<L.nb_cell, kThreads, 0, ST>>>(L, W.table, W.tiles, W.ids, faces);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
